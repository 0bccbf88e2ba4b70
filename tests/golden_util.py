"""Loading helpers for the reference-generated fixtures under tests/golden/ (see
tests/golden/make_reference_vectors.py for how they were produced)."""
import glob
import io
import os

import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def unpack_state_dict(sd):
    """Inverse of make_reference_vectors.pack_state_dict: densify the (shape, idx, val) `w3j` records."""
    out = {}
    for k, v in sd.items():
        if isinstance(v, dict):
            t = torch.zeros(v["w3j_shape"], dtype=v["dtype"])
            t[tuple(v["idx"].long().T)] = v["val"]
            out[k] = t
        else:
            out[k] = v
    return out


SHARD_BYTES = 900_000  # every fixture file stays under 1 MB


def save_sharded(obj, stem):
    """Write a list of records (or a dict of such lists) as tests/golden/<stem>.<i>.pt shards of at most SHARD_BYTES each;
    load_sharded(stem) restores the object."""
    items = [(k, r) for k, v in obj.items() for r in v] if isinstance(obj, dict) else [(None, r) for r in obj]

    def pack(part):
        if isinstance(obj, dict):
            return {k: [r for kk, r in part if kk == k] for k in obj}
        return [r for _, r in part]

    def nbytes(part):
        buf = io.BytesIO()
        torch.save(pack(part), buf)
        return buf.tell()

    for f in glob.glob(os.path.join(GOLDEN, f"{stem}.*.pt")):
        os.remove(f)
    shards, cur = [], []
    for it in items:
        if cur and nbytes(cur + [it]) > SHARD_BYTES:
            shards.append(cur)
            cur = []
        cur.append(it)
    shards.append(cur)
    for i, part in enumerate(shards):
        torch.save(pack(part), os.path.join(GOLDEN, f"{stem}.{i}.pt"))
    return len(shards)


def load_sharded(stem):
    files = sorted(glob.glob(os.path.join(GOLDEN, f"{stem}.*.pt")), key=lambda f: int(f.rsplit(".", 2)[1]))
    parts = [torch.load(f, weights_only=False) for f in files]
    if isinstance(parts[0], dict):
        return {k: [r for p in parts for r in p[k]] for k in parts[0]}
    return [r for p in parts for r in p]


def load_models():
    return load_sharded("ref_models")


def load_ops():
    return load_sharded("ref_ops")


def model_case_ids():
    return [r["name"] for r in load_models()]
