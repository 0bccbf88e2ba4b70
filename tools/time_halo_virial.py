"""Cost of the stress / per-atom virial / heat-current outputs of the multi-GPU step (run under torchrun, one rank per GPU):

    torchrun --nproc_per_node N tools/time_halo_virial.py [--rounds 7] [--steps 50]

c2 replicated N x along x (as bench.py --gpus N), fp32, P2P halo, one CUDA graph per configuration: off, stress, atomic
virial, heat current.  The configurations are replayed in alternation over rounds and the median ms per step of each
(max over ranks) is printed by rank 0.  Then the new halo pieces are timed eagerly against the ones they replace: the
width-12 reverse rows against the width-3 ones and the 13-value all-reduce against the energy all-reduce (CUDA events
around each call, after a forward halo that starts the step)."""
import argparse
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from allegro_b200 import systems  # noqa: E402
from allegro_b200.halo import DistributedAllegro, GraphedDistributedAllegro, P2PHalo, SlabDecomposition  # noqa: E402
from allegro_b200.model import AllegroModel  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=7)
ap.add_argument("--steps", type=int, default=50)
args = ap.parse_args()

rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]))
torch.cuda.set_device(dev)
dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
pos, cell, types = systems.make_positions("c2", (14 * world, 14, 14))
dec = SlabDecomposition(pos, cell, types, systems.CONFIGS["c2"]["r_max"], rank, world, device=dev)
cnt = torch.tensor([float(dec.n_edges), float(dec.n_owned)], device=dev, dtype=torch.float64)
dist.all_reduce(cnt)
model = AllegroModel(**systems.model_kwargs("c2", float(cnt[0] / cnt[1]), "float32")).to(dev).model
po = dec.local_positions_from_global(pos)[: dec.n_owned].to(dev, torch.float32)
vel = torch.randn(po.shape, generator=torch.Generator().manual_seed(rank), dtype=torch.float32).to(dev)
dec.to(dev)
p2p = P2PHalo(dec, dev, atomic_virial=True)
plain = P2PHalo(dec, dev)

CONFIGS = {"off": dict(), "stress": dict(stress=True), "atomic_virial": dict(atomic_virial=True), "heat_current": dict(heat_current=True)}
graphs = {}
for name, fl in CONFIGS.items():
    runner = DistributedAllegro(model, dec, p2p=p2p if fl else plain, **fl)
    graphs[name] = GraphedDistributedAllegro(runner, po, velocities=vel)


def timed(fn, steps):
    dist.barrier()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    t = torch.tensor([a.elapsed_time(b) / steps], device=dev, dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)


ms = {k: [] for k in CONFIGS}
for name in CONFIGS:  # warm-up
    timed(graphs[name], 5)
for _ in range(args.rounds):
    for name in CONFIGS:
        ms[name].append(timed(graphs[name], args.steps))

# eager per-call times of the new halo pieces (a forward halo starts every step: it bumps the step number)
n, nl = dec.n_owned, dec.n_owned + dec.n_ghost
g = torch.randn(nl, 3, device=dev)
W = torch.randn(nl, 3, 3, device=dev)
go, Wo = torch.zeros(n, 3, device=dev), torch.zeros(n, 3, 3, device=dev)
e1, v13 = torch.zeros(1, device=dev, dtype=torch.float64), torch.zeros(13, device=dev, dtype=torch.float64)
pieces = {"reverse (width 3)": lambda: p2p.reverse(g, go), "reverse_w (width 12)": lambda: p2p.reverse_w(g, W, go, Wo),
          "energy all-reduce (1)": lambda: p2p.energy(e1), "vector all-reduce (13)": lambda: p2p.reduce(v13)}
eager = {k: [] for k in pieces}
for _ in range(args.rounds):
    for name, fn in pieces.items():
        for _ in range(args.steps):
            p2p.forward(po)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            eager[name].append(a.elapsed_time(b))
if rank == 0:
    print(f"c2 x{world}: {pos.shape[0]} atoms, {dec.n_owned} owned + {dec.n_ghost} ghosts on rank 0, fp32, P2P, graph replay")
    for name in CONFIGS:
        print(f"  {name:16s} {statistics.median(ms[name]):8.3f} ms/step   (rounds: {' '.join(f'{x:.3f}' for x in ms[name])})")
    print("  halo bytes/step/rank: %d without W rows, %d with" % (dec.halo_bytes_per_step(8), dec.halo_bytes_per_step(8, atomic_virial=True)))
    for name, t in eager.items():
        print(f"  eager {name:24s} {statistics.median(t) * 1e3:8.1f} us")
    print(f"  P2P error word: {p2p.error()}")
dist.barrier()
torch.cuda.synchronize()
os._exit(0)  # live graphs: leave without the destructors
