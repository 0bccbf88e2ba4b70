"""Molecular dynamics on several GPUs with DistributedCalculator (run under torchrun, one rank per GPU):

    torchrun --nproc_per_node N tools/time_slab_md.py [--steps 300] [--dt 1.0] [--temperature 300] [--basis cubic,tilted]

c2 replicated N x along x (as bench.py --gpus N), fp32, P2P halo, r_max + skin = 5.5 A, velocities drawn from the
Maxwell-Boltzmann distribution at --temperature for Cu, velocity Verlet at --dt fs.  With more ranks than devices the
ranks share the devices round-robin (gloo for set-up and migration; the per-step path is the P2P mailboxes either way),
so two ranks on one H100 is allowed, and its numbers include the two processes contending for one GPU.

Rank 0 prints one JSON line: MD ns/day including rebuilds, mean steps between rebuilds, the mean rebuild time split into
plan, migration, ghost exchange, neighbour list and graph capture (wall time, max over ranks), the step time of the
static GraphedDistributedAllegro on the same first frame, and the card name and power limit.

--basis: ``cubic`` (the default) is the orthorhombic box; ``tilted`` is the same atoms in the rows (a, b + a, c) of the
same crystal (slabs with slanted faces, H_0 = |a| |b| / |a + b|, the 14 world replicas along a keep H_0 / world >=
r_max + skin up to world 8), which takes the lattice kernels (ab2_slab_plan_count_lattice, ab2_p2p_push_rows_v).  A comma-separated
list runs the bases alternately, --rounds times each, in one call; one JSON line per run."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from allegro_b200 import systems  # noqa: E402
from allegro_b200.halo import DistributedAllegro, DistributedCalculator, GraphedDistributedAllegro, P2PHalo, SlabDecomposition  # noqa: E402
from allegro_b200.model import AllegroModel  # noqa: E402

AMU = 103.6427  # eV fs^2 / A^2
KB = 8.617333e-5  # eV / K

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=300)
ap.add_argument("--dt", type=float, default=1.0)
ap.add_argument("--temperature", type=float, default=300.0)
ap.add_argument("--skin", type=float, default=0.5)
ap.add_argument("--basis", default="cubic", help="cubic, tilted, or a comma-separated list run alternately")
ap.add_argument("--rounds", type=int, default=1, help="runs of every basis (alternating)")
args = ap.parse_args()
bases = args.basis.split(",")
if not set(bases) <= {"cubic", "tilted"}:
    ap.error(f"--basis: cubic or tilted, got {args.basis!r}")

rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
ndev = torch.cuda.device_count()
dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]) % ndev)
torch.cuda.set_device(dev)
shared = world > ndev
if shared:
    dist.init_process_group("gloo", rank=rank, world_size=world)
else:
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)


def max_over_ranks(v: float) -> float:
    t = torch.tensor([v], dtype=torch.float64, device="cpu" if shared else dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t[0])


r_max = systems.CONFIGS["c2"]["r_max"]
mass = 63.546


def frame(basis):
    """(pos, rows, types): c2 (14 world, 14, 14) in its cubic box, or (tilted) the same atoms in the rows (a, b + a, c):
    slanted faces, H_0 = |a| |b| / |a + b| (>= 6.3 A per rank up to world 8)"""
    pos, cell, types = systems.make_positions("c2", (14 * world, 14, 14))
    if basis == "tilted":
        A, B, C = cell
        cell = torch.stack([A, B + A, C])
    return pos, cell, types


def run(basis):
    pos, cell, types = frame(basis)
    g = torch.Generator().manual_seed(0)
    vel = torch.randn(pos.shape, generator=g, dtype=torch.float64) * (KB * args.temperature / (mass * AMU)) ** 0.5
    vel -= vel.mean(0)

    # static step on the first frame (the reference point: no rebuild check, plain mailbox)
    dec = SlabDecomposition(pos, cell, types, r_max, rank, world, device=dev)
    cnt = torch.tensor([float(dec.n_edges), float(dec.n_owned)], dtype=torch.float64, device="cpu" if shared else dev)
    dist.all_reduce(cnt)
    model = AllegroModel(**systems.model_kwargs("c2", float(cnt[0] / cnt[1]), "float32")).to(dev).model
    po = dec.local_positions_from_global(pos)[: dec.n_owned].to(dev, torch.float32)
    dec.to(dev)
    static_p2p = P2PHalo(dec, dev)
    static = GraphedDistributedAllegro(DistributedAllegro(model, dec, p2p=static_p2p), po)

    def timed_replays(n):
        dist.barrier()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            static()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / n

    timed_replays(10)
    static_ms = max_over_ranks(min(timed_replays(50) for _ in range(3)))
    del static
    static_p2p.close()

    # the trajectory
    calc = DistributedCalculator(model, cell, r_max, args.skin, rank, world, device=dev, transport="p2p")
    t0 = time.perf_counter()
    local = calc.distribute(pos.to(torch.float32), types, velocities=vel.to(torch.float32), masses=torch.full((pos.shape[0],), mass))
    torch.cuda.synchronize()
    setup_s = time.perf_counter() - t0
    for k in calc.rebuild_seconds:
        calc.rebuild_seconds[k] = 0.0
    first = calc.n_rebuilds
    out = calc.compute(local)
    dist.barrier()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        inv_m = 1.0 / (local.arrays["masses"][:, None] * AMU)
        local.arrays["velocities"] += 0.5 * args.dt * out["forces"] * inv_m
        local.pos += args.dt * local.arrays["velocities"]
        out = calc.compute(local)
        inv_m = 1.0 / (local.arrays["masses"][:, None] * AMU)
        local.arrays["velocities"] += 0.5 * args.dt * out["forces"] * inv_m
    torch.cuda.synchronize()
    wall = max_over_ranks(time.perf_counter() - t0)
    n_rebuilds = calc.n_rebuilds - first
    split = {k: max_over_ranks(v / max(n_rebuilds, 1)) * 1e3 for k, v in calc.rebuild_seconds.items()}
    n_owned = max_over_ranks(float(len(local)))
    lattice = not calc.geom.diagonal
    calc.close()

    if rank == 0:
        try:
            power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(dev.index)],
                                   capture_output=True, text=True, timeout=30).stdout.strip()
        except (OSError, subprocess.SubprocessError):
            power = "unknown"
        print(json.dumps({
            "basis": basis, "lattice_kernels": lattice, "world": world, "ranks_per_device": -(-world // ndev), "atoms": int(pos.shape[0]),
            "max_owned_atoms": int(n_owned), "steps": args.steps, "dt_fs": args.dt, "temperature_K": args.temperature, "skin": args.skin,
            "md_ns_per_day": args.steps * args.dt * 1e-6 / wall * 86400.0, "md_ms_per_step": wall / args.steps * 1e3,
            "rebuilds": n_rebuilds, "mean_steps_between_rebuilds": args.steps / n_rebuilds if n_rebuilds else None,
            "rebuild_ms": split, "rebuild_ms_total": sum(split.values()), "setup_s": setup_s,
            "static_graphed_step_ms": static_ms, "gpu": torch.cuda.get_device_name(dev), "power_limit": power,
        }), flush=True)


for _ in range(args.rounds):
    for basis in bases:
        run(basis)
dist.barrier()
dist.destroy_process_group()
