"""fp32 models across the architecture grid against the fp64 oracle, with the dispatch of the fused kernels checked.

The fused MLP kernels (ab2_mlp2, ab2_mlp2_readout) and the composed tensor products (ab2_tp_chain_fwd / _bwd) are chosen
at run time: the library takes or declines each call from its shapes and a shared-memory plan, and AllegroCore /
PackedMLP run a slower path when it declines.  Each case here builds the fp32 AllegroModel and the fp64 AllegroOracle from
one state dict (test_gpu_model._pair) and compares atomic energies, total energy and forces at the fp32 bar (1e-4).  Spies
on the four entries record, per stage tag, which entry was asked and whether it took the call; the record must equal
DISPATCH below, so that no case passes on a fallback it was not meant to take.  Spies on ab2_tp_fwd / ab2_tp_bwd check
that the stored-feature tensor products run, once per layer and direction, exactly when the composed ones do not.  (The
kernel families behind ab2_tp_fwd / ab2_tp_bwd are checked per table with torch.profiler in test_gpu_tp_ragged; more
profiler sessions over whole models in the same pytest process made those traces lose kernel records.)
"""
import pytest
import torch

from allegro_b200 import _lib
from allegro_b200 import data as D
from allegro_b200.model import AllegroModel
from oracle.model_ref import AllegroOracle
from test_gpu_model import _check, _pair

pytestmark = pytest.mark.gpu

TOL = 1e-4
# l_max = 3 in fp32 runs the shape-generic tensor-product kernels (tp.cu) on a 353-entry layer-0 table, with fp32
# atomics; the same templates meet 1e-9 in fp64 (test_gpu_model.test_c5_lmax3_three_layers_fp64).  Measured force
# errors on an H100: 1.25e-4 (3^3 cell) and 1.13e-4 (5^3 cell) of max |F|; energies meet 1e-4.
# l_max 4 runs the same generic kernels on tables of 1158 (L = 2) and 2052 entries (L = 3); measured on an H100 (700 W) at
# 3^3 in two runs: forces 2.55e-5 / 2.60e-5 (L = 2) and 7.68e-5 / 8.11e-5 (L = 3) of max |F|, energies 3.1e-5 / 2.4e-5.
# The bars are 1.5x the larger measurement.  The same fp32 models
# through the host pipeline with the kernels' torch restatement in fp32 on the CPU (tests/kernel_spec.py) land at 5.7e-6 /
# 1.3e-5: the CUDA error is 5-9x that at every l_max (lmax0, lmax1 and lmax3 alike), so it is not the l_max 4 tables.
TOL_F = {"lmax3": 2e-4, "lmax4": 4e-5, "lmax4_L3": 1.2e-4}

# c2 widths (S = H = readout hidden width = 64, U = 32, l_max = 2, L = 2), then per case the overrides
C3_AT_C2_WIDTHS = dict(num_scalar_features=64, num_tensor_features=32, radial_chemical_embed_dim=64, scalar_embed_mlp_hidden_layers_width=64,
                       allegro_mlp_hidden_layers_width=64, readout_mlp_hidden_layers_width=64)
CASES = {
    "L1_U32": dict(num_layers=1),
    "L1_U64": dict(num_layers=1, num_tensor_features=64),
    "L1_U96": dict(num_layers=1, num_tensor_features=96),
    "L1_U128": dict(num_layers=1, num_tensor_features=128),
    "L2_U32": dict(),
    "L2_U64": dict(num_tensor_features=64),
    "L2_U96": dict(num_tensor_features=96),
    "L3_U32": dict(num_layers=3),
    "L3_U64": dict(num_layers=3, num_tensor_features=64),
    "S32": dict(num_scalar_features=32, radial_chemical_embed_dim=32, scalar_embed_mlp_hidden_layers_width=32, allegro_mlp_hidden_layers_width=32,
                readout_mlp_hidden_layers_width=32),
    "lmax1": dict(l_max=1),
    "lmax3": dict(l_max=3),
    "no_coupling": dict(tp_path_channel_coupling=False),
    "deep_mlps": dict(allegro_mlp_hidden_layers_depth=2, readout_mlp_hidden_layers_depth=2),
    "linear_latents": dict(allegro_mlp_nonlinearity=None),
    "three_species": dict(C3_AT_C2_WIDTHS, per_type_energy_scales=[2.5, 0.5, 1.25], per_type_energy_shifts=[-1.25, 0.5, 2.0],
                          per_edge_type_cutoff={"Li": 4.0, "P": {"Li": 5.0, "P": 4.5, "S": 6.0}, "S": 5.5}),
    "lmax0": dict(l_max=0),
    "lmax4": dict(l_max=4),
    "lmax4_L3": dict(l_max=4, num_layers=3),
}

# Which entry each stage asks, in call order, and its verdict: "+" taken, "-" declined (the caller then runs the separate
# MLPs or the plain linear layers).  mlp2 = ab2_mlp2, ro = ab2_mlp2_readout, chain / chain_bwd = ab2_tp_chain_fwd / _bwd.
# The byte counts are the shared-memory plans of linear_tc.cu at the H100's 232 448-byte opt-in limit (the smallest
# plan, 2 raw slots and 2 stages, where a call is declined); "K x H -> N" the shape of an ab2_mlp2 call.
#   ab2_mlp2_readout takes (L, U) = (1, 32..128) and (2, 32) in both directions; (2, 64) needs 235 648 / 234 624 bytes,
#   (2, 96) 243 840 / 242 816, (3, 32) 260 224 / 259 200, (3, 64) 268 416 / 267 392; H = 32 is not built (RO_H = 64).
#   ab2_mlp2 takes every stage except: N > 256 (more than four 64-column chunks), and 192 x 64 -> 256 / 256 x 64 -> 192
#   (235 520 bytes), 352 x 64 -> 160 (251 904 bytes).
#   ab2_tp_chain_*: two-layer l_max = 2 models with the baked tables, U = 32 or 64, E > 0.
C2 = {  # L = 2, U = 32 (c2): composed tensor products, fused readout
    "fwd.L0": "chain+ mlp2+",          # 96 x 64 -> 160: 219 136 bytes
    "fwd.L1": "chain+ ro+",            # 227 456 bytes
    "bwd.readout": "ro+",              # 226 432 bytes
    "bwd.L1": "chain_bwd+",
    "bwd.L0": "mlp2+ chain_bwd+",      # 160 x 64 -> 96
}
L1 = {"fwd.L0": "ro+", "bwd.readout": "ro+"}  # P = 64: the last latent MLP is the only one
DISPATCH = {
    "L1_U32": L1, "L1_U64": L1, "L1_U96": L1, "L1_U128": L1,
    "L2_U32": C2,
    "L2_U64": {
        "fwd.L0": "chain+ mlp2+",      # 128 x 64 -> 256 (four chunks): 219 136 bytes
        "fwd.L1": "chain+ ro- mlp2+",  # ro: 235 648 bytes; 192 x 64 -> 64
        "fwd.readout": "mlp2+",        # 192 x 64 -> 1
        "bwd.readout": "ro- mlp2+",    # ro: 234 624 bytes; rank-1 1 x 64 -> 192
        "bwd.L1": "mlp2+ chain_bwd+",  # 64 x 64 -> 192
        "bwd.L0": "mlp2+ chain_bwd+",  # 256 x 64 -> 128: 219 136 bytes
    },
    "L2_U96": {  # U = 96: no composed tensor products
        "fwd.L0": "mlp2-",             # 160 x 64 -> 352: six chunks
        "fwd.L1": "ro- mlp2+",         # ro: 243 840 bytes; 224 x 64 -> 64
        "fwd.readout": "mlp2+",
        "bwd.readout": "ro- mlp2+",    # ro: 242 816 bytes
        "bwd.L1": "mlp2+",             # 64 x 64 -> 224
        "bwd.L0": "mlp2-",             # 352 x 64 -> 160: 251 904 bytes
    },
    "L3_U32": {
        "fwd.L0": "mlp2+", "fwd.L1": "mlp2+",  # 96 x 64 -> 160, 160 x 64 -> 160 (202 752 bytes)
        "fwd.L2": "ro- mlp2+",         # ro: 260 224 bytes; 224 x 64 -> 64
        "fwd.readout": "mlp2+",        # 256 x 64 -> 1
        "bwd.readout": "ro- mlp2+",    # ro: 259 200 bytes; rank-1 1 x 64 -> 256
        "bwd.L2": "mlp2+", "bwd.L1": "mlp2+", "bwd.L0": "mlp2+",
    },
    "L3_U64": {
        "fwd.L0": "mlp2+",             # 128 x 64 -> 256
        "fwd.L1": "mlp2-",             # 192 x 64 -> 256: 235 520 bytes
        "fwd.L2": "ro- mlp2+",         # ro: 268 416 bytes
        "fwd.readout": "mlp2+",
        "bwd.readout": "ro- mlp2+",    # ro: 267 392 bytes
        "bwd.L2": "mlp2+",             # 64 x 64 -> 256
        "bwd.L1": "mlp2-",             # 256 x 64 -> 192: 235 520 bytes
        "bwd.L0": "mlp2+",             # 256 x 64 -> 128
    },
    "S32": {  # S = H = 32: the readout is fused on the host (equal hidden widths), the library declines H = 32
        "fwd.L0": "chain+ mlp2+",      # 64 x 32 -> 128
        "fwd.L1": "chain+ ro- mlp2+",  # 96 x 32 -> 32
        "fwd.readout": "mlp2+",        # 96 x 32 -> 1
        "bwd.readout": "ro- mlp2+",    # rank-1 1 x 32 -> 96
        "bwd.L1": "mlp2+ chain_bwd+",
        "bwd.L0": "mlp2+ chain_bwd+",
    },
    # l_max = 1 and 3 have no composed tensor products (D != 9); their first latent MLPs: 96 x 64 -> 128 and -> 192
    "lmax1": {"fwd.L0": "mlp2+", "fwd.L1": "ro+", "bwd.readout": "ro+", "bwd.L0": "mlp2+"},
    "lmax3": {"fwd.L0": "mlp2+", "fwd.L1": "ro+", "bwd.readout": "ro+", "bwd.L0": "mlp2+"},
    "no_coupling": C2,  # the same tables; the coupling weights are broadcast over the channels
    # three-layer MLPs: no ab2_mlp2 and no fused readout
    "deep_mlps": {"fwd.L0": "chain+", "fwd.L1": "chain+", "bwd.L1": "chain_bwd+", "bwd.L0": "chain_bwd+"},
    # linear latent MLPs: no ab2_mlp2 for them, no fused readout (the last latent MLP is not SiLU); the readout's own
    "linear_latents": {"fwd.L0": "chain+", "fwd.L1": "chain+", "fwd.readout": "mlp2+", "bwd.readout": "mlp2+",
                       "bwd.L1": "chain_bwd+", "bwd.L0": "chain_bwd+"},
    "three_species": C2,
    # l_max 0 and 4: no composed tensor products either; the env weights are (l_max + 1) U wide, so the first latent MLP is
    # 96 x 64 -> 96 and 96 x 64 -> 224 (S + 5U, under the four-chunk limit) and its backward 96 / 224 x 64 -> 96; the fused
    # readout depends on (L, U) only: taken at (2, 32), declined at (3, 32) as in L3_U32
    "lmax0": {"fwd.L0": "mlp2+", "fwd.L1": "ro+", "bwd.readout": "ro+", "bwd.L0": "mlp2+"},
    "lmax4": {"fwd.L0": "mlp2+", "fwd.L1": "ro+", "bwd.readout": "ro+", "bwd.L0": "mlp2+"},
    "lmax4_L3": {
        "fwd.L0": "mlp2+", "fwd.L1": "mlp2+",  # both write S + 5U = 224 columns
        "fwd.L2": "ro- mlp2+",         # ro: 260 224 bytes; 224 x 64 -> 64
        "fwd.readout": "mlp2+",
        "bwd.readout": "ro- mlp2+",    # ro: 259 200 bytes
        "bwd.L2": "mlp2+", "bwd.L1": "mlp2+", "bwd.L0": "mlp2+",
    },
}
# A frame without edges: the direct path, and the torch.autograd path (use_autograd), return zeros before any kernel
NO_EDGES_AUTOGRAD = {"L2_U32": {}, "L1_U32": {}}

SPIED = {"mlp2": "mlp2", "mlp2_readout": "ro", "tp_chain_fwd": "chain", "tp_chain_bwd": "chain_bwd"}


def _frames(case):
    if case == "three_species":
        return ["c3_4", "c3_6"]
    frames = ["c2_3", "c2_5"] if not case.startswith("lmax4") else ["c2_3"]  # the fp64 oracle at l_max 4 takes ~20 s at 3^3
    if case in NO_EDGES_AUTOGRAD:
        frames += ["isolated_atoms_ragged_rows", "no_edges_at_all"]
    return frames


def _cases():
    return [pytest.param(c, f, id=f"{c}-{f}") for c in CASES for f in _frames(c)]


def _spy(monkeypatch):
    """Wrap the four entries with call-through spies; returns the record [(stage tag, entry, taken)]."""
    rec = []
    for fn, short in SPIED.items():
        real = getattr(_lib, fn)

        def spy(*a, _real=real, _short=short, **k):
            ok = _real(*a, **k)
            rec.append((_lib._TAG[0], _short, bool(ok)))
            return ok

        monkeypatch.setattr(_lib, fn, spy)
    return rec


def _dispatch(rec):
    out = {}
    for tag, entry, ok in rec:
        out[tag] = (out[tag] + " " if tag in out else "") + entry + ("+" if ok else "-")
    return out


def _golden_pair(name, over):
    """Oracle and fp32 model on the frame of a golden case (two species, open boundaries, r_max 3.5)."""
    from allegro_b200 import systems
    from golden_util import load_models

    d = dict({r["name"]: r for r in load_models()}[name]["data"])
    kw = systems.model_kwargs("c2", 9.0, "float64")
    kw.update(type_names=["X", "Y"], r_max=3.5, per_type_energy_shifts=[0.5, -1.0])
    kw.update(over)
    oracle = AllegroOracle(**kw)
    model = AllegroModel(**dict(kw, model_dtype="float32"))
    model.load_state_dict(oracle.state_dict())
    return oracle, model.to("cuda"), d


def _spy_tp(monkeypatch):
    """Call-through spies on the stored-feature tensor products; returns the record [(entry, stage tag)]."""
    rec = []
    for fn in ("tp_fwd", "tp_bwd"):
        real = getattr(_lib, fn)

        def spy(*a, _real=real, _fn=fn, **k):
            rec.append((_fn, _lib._TAG[0]))
            return _real(*a, **k)

        monkeypatch.setattr(_lib, fn, spy)
    return rec


@pytest.mark.parametrize("case,frame", _cases())
def test_fp32_grid(case, frame, monkeypatch):
    over = CASES[case]
    if frame.startswith(("c2_", "c3_")):
        name, scale = frame.split("_")
        oracle, model, d = _pair(name, int(scale), "float32", **over)
    else:
        oracle, model, d = _golden_pair(frame, over)
    E = d[D.EDGE_INDEX_KEY].shape[1]
    rec, tp_rec = _spy(monkeypatch), _spy_tp(monkeypatch)
    ee, ef = _check(oracle, model, d, TOL, TOL_F.get(case, TOL))
    got = _dispatch(rec)
    print(f"\n{case} {frame} (E = {E}): E {ee:.2e} F {ef:.2e}  dispatch {got}")
    core = model.model.core()
    assert got == (DISPATCH[case] if E else {})
    if E == 0:
        assert tp_rec == []
        rec.clear()
        model.use_autograd = True
        try:
            ee, ef = _check(oracle, model, d, TOL, TOL)
        finally:
            model.use_autograd = False
        got = _dispatch(rec)
        print(f"  through torch.autograd: E {ee:.2e} F {ef:.2e}  dispatch {got}")
        assert got == NO_EDGES_AUTOGRAD[case]
        return
    # the stored-feature tensor products: every layer forward, then backward from the last layer, unless composed
    L = len(core.layers)
    stored = [("tp_fwd", f"fwd.L{l}") for l in range(L)] + [("tp_bwd", f"bwd.L{l}") for l in range(L - 1, -1, -1)]
    assert tp_rec == ([] if core.chain is not None else stored), tp_rec
