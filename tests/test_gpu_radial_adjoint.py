"""The scalar-embed MLP's hidden-gradient GEMM with the radial adjoint as its epilogue (ab2_radial_pq_bwd_gemm, reached
through ``_lib.radial_pq_bwd(..., gemm=...)``) on the H100:

- against the two launches it replaces (``_lib.linear`` for g_h = Gout @ W2^T, then ``_lib.radial_pq_bwd`` with aux = h)
  on identical inputs: ragged row counts, one to three species with a per-pair cutoff table, edges beyond their pair's
  cutoff and within an ulp of it, every nonlinearity, hidden widths 64 and 32, a strided middle gradient segment (as
  gX[:, :S] is) and gvec pre-filled;
- the cases it declines: nothing computed, gvec untouched, and a model then takes the two launches;
- a c2-architecture model, which takes the fused kernel, against the fp64 oracle.
"""
import math

import pytest
import torch

from allegro_b200 import _lib
from allegro_b200 import data as D
from allegro_b200 import systems
from allegro_b200.model import AllegroModel
from oracle.model_ref import AllegroOracle
from test_gpu_model import _check, _pair

pytestmark = pytest.mark.gpu

DEV = "cuda"
NLS = {"silu": _lib.NL_SILU, "mish": _lib.NL_MISH, "gelu": _lib.NL_GELU}
P_CUT = 6.0
N_ATOMS = 500
SEG = (96, 64, 96)  # [gw0 | gX[:, :S] | gomega] of the c2 architecture: K = 256
LD_MID = 192        # row stride of the strided middle segment (X holds S (L + 1) columns)


def _inputs(M, T, H, seed, dtype=torch.float32, seg=SEG):
    """Operands of one radial adjoint: edge geometry with a per-pair cutoff table, PQ, the gradient segments and W2^T."""
    g = torch.Generator().manual_seed(seed)
    types = torch.randint(0, T, (N_ATOMS,), generator=g, dtype=torch.int32)
    ctr = torch.randint(0, N_ATOMS, (M,), generator=g, dtype=torch.int32)
    nbr = torch.randint(0, N_ATOMS, (M,), generator=g, dtype=torch.int32)
    rmax = 4.0 + 0.5 * torch.arange(T, dtype=torch.float32).view(-1, 1) + 0.25 * torch.arange(T, dtype=torch.float32).view(1, -1)
    pair = (types[ctr.long()] * T + types[nbr.long()]).long()
    rm = rmax.reshape(-1)[pair]
    u = torch.randn(M, 3, generator=g, dtype=torch.float64)
    u = u / u.norm(dim=1, keepdim=True)
    r = (0.25 + 1.0 * torch.rand(M, generator=g, dtype=torch.float64)) * rm.double()  # about 1 in 5 beyond the pair's cutoff
    vec = (u * r.view(-1, 1)).float()
    # edges along an axis at the cutoff, one float below it and one above: |vec| is then exact and x = |r| / r_max is
    # 1 - ulp, exactly 1 and 1 + ulp
    k = min(M, 6)
    for i in range(k):
        rr = rm[i].reshape(1)
        step = torch.tensor([-math.inf, math.inf, -math.inf, 0.0, math.inf, 0.0][i], dtype=torch.float32).reshape(1)
        edge = rr if step == 0 else torch.nextafter(rr, step)
        vec[i] = 0.0
        vec[i, i % 3] = edge[0] * (1 if i % 2 else -1)
    bw = torch.arange(1, 9, dtype=torch.float32) * math.pi
    PQ = torch.randn(T * T, 8, H, generator=g, dtype=torch.float32) / 2
    K = sum(seg)
    WT = (torch.randn(K, H, generator=g, dtype=torch.float64) / math.sqrt(K)).float()
    gw0 = torch.randn(M, seg[0], generator=g, dtype=torch.float32)
    X = torch.randn(M, LD_MID, generator=g, dtype=torch.float32)
    gom = torch.randn(M, seg[2], generator=g, dtype=torch.float32)
    gvec0 = torch.randn(M, 3, generator=g, dtype=torch.float32)
    dev = lambda t: t.to(DEV, dtype) if t.is_floating_point() else t.to(DEV)
    X = dev(X)
    gouts = [dev(gw0), X[:, : seg[1]], dev(gom)]
    f32 = lambda t: t.to(DEV)
    return dict(vec=f32(vec), ctr=dev(ctr), nbr=dev(nbr), types=dev(types), rmax=f32(rmax), bw=f32(bw), PQ=f32(PQ), WT=dev(WT), gouts=gouts,
                gvec0=f32(gvec0), H=H)


def _two_launches(a, nl):
    """What the model ran before the fused kernel: g_h = Gout @ W2^T, h = the radial kernel's output, then the adjoint."""
    dt = a["gouts"][0].dtype
    M = a["vec"].shape[0]
    h = _lib.radial_pq_fwd(dt, a["H"], P_CUT, a["vec"], a["ctr"], a["nbr"], a["types"], a["rmax"], a["bw"], a["PQ"])
    g_h = torch.empty(M, a["H"], dtype=dt, device=DEV)
    _lib.linear(a["gouts"], a["WT"], [g_h], W_packed=_lib.linear_pack(a["WT"]))
    gvec = a["gvec0"].clone()
    _lib.radial_pq_bwd(dt, a["H"], P_CUT, a["vec"], a["ctr"], a["nbr"], a["types"], a["rmax"], a["bw"], a["PQ"], g_h, h, gvec, nonlin=nl)
    return gvec, h


def _fused(a, nl, h):
    dt = a["gouts"][0].dtype
    gvec = a["gvec0"].clone()
    ok = _lib.radial_pq_bwd(dt, a["H"], P_CUT, a["vec"], a["ctr"], a["nbr"], a["types"], a["rmax"], a["bw"], a["PQ"], None, h, gvec, nonlin=nl,
                            gemm=(a["gouts"], _lib.linear_pack(a["WT"])))
    return ok, gvec


CASES = ([(M, 3, "silu", 64) for M in (1, 127, 128, 129, 4097, 200003)]
         + [(4097, T, nl, 64) for T in (1, 2, 3) for nl in NLS]
         + [(4097, 3, nl, 32) for nl in NLS])


@pytest.mark.parametrize("M,T,nl,H", CASES)
def test_fused_matches_two_launches(M, T, nl, H):
    a = _inputs(M, T, H, seed=M + 10 * T + H)
    ref, h = _two_launches(a, NLS[nl])
    ok, got = _fused(a, NLS[nl], h)
    assert ok
    inc = ref - a["gvec0"]
    assert bool(torch.isfinite(got).all())
    err = float((got - ref).abs().max() / inc.abs().max().clamp_min(1e-30))
    assert err <= 1e-5, err
    # one writer per row, no atomics: a second launch gives the same bits
    ok2, again = _fused(a, NLS[nl], h)
    assert ok2 and torch.equal(got, again)
    # the edges at and beyond their pair's cutoff receive nothing
    r = a["vec"].norm(dim=1)
    pair = (a["types"][a["ctr"].long()] * T + a["types"][a["nbr"].long()]).long()
    out = r >= a["rmax"].reshape(-1)[pair]
    assert torch.equal(got[out], a["gvec0"][out])


def test_zero_rows():
    a = _inputs(1, 1, 64, seed=1)
    gvec = torch.empty(0, 3, device=DEV)
    e = torch.empty(0, dtype=torch.int32, device=DEV)
    segs = [t[:0] for t in a["gouts"]]
    assert _lib.radial_pq_bwd(torch.float32, 64, P_CUT, a["vec"][:0], e, e, a["types"], a["rmax"], a["bw"], a["PQ"], None,
                              torch.empty(0, 64, device=DEV), gvec, gemm=(segs, _lib.linear_pack(a["WT"])))


DECLINES = {
    "bf16": dict(dtype=torch.bfloat16),
    "fp64": dict(dtype=torch.float64),
    "hidden_128": dict(H=128),
    "pq_beyond_smem": dict(T=4),                 # 4^2 x 8 x 64 floats = 32 KB
    "segment_not_32_wide": dict(seg=(80, 64, 112)),
    "segment_misaligned": dict(offset=1),        # middle segment X[:, 1:65]: not 16-byte aligned
}


@pytest.mark.parametrize("case", list(DECLINES))
def test_declines(case):
    c = dict(dtype=torch.float32, H=64, T=2, seg=SEG, offset=0)
    c.update(DECLINES[case])
    a = _inputs(1000, c["T"], c["H"], seed=5, dtype=c["dtype"], seg=c["seg"])
    if c["offset"]:
        X = a["gouts"][1]
        a["gouts"][1] = X.as_strided(X.shape, X.stride(), X.storage_offset() + c["offset"])
    dt = c["dtype"]
    # (an fp32 image for every dtype, so that the entry itself, not the missing image, declines)
    h = torch.zeros(1000, c["H"], dtype=dt, device=DEV)
    gvec = a["gvec0"].to(_lib.ACC_DTYPE[dt]).clone()
    before = gvec.clone()
    n0 = _lib.PROF.launches
    ok = _lib.radial_pq_bwd(dt, c["H"], P_CUT, gvec.new_tensor(a["vec"]), a["ctr"], a["nbr"], a["types"], gvec.new_tensor(a["rmax"]),
                            gvec.new_tensor(a["bw"]), gvec.new_tensor(a["PQ"]), None, h, gvec, gemm=(a["gouts"], _lib.linear_pack(a["WT"].float())))
    torch.cuda.synchronize()
    assert ok is False
    assert torch.equal(gvec, before)
    assert _lib.PROF.launches == n0  # a declined call is not counted as a launch


def test_unknown_nonlinearity_is_an_error():
    a = _inputs(100, 1, 64, seed=2)
    with pytest.raises(RuntimeError, match="nonlinearity"):
        _lib.radial_pq_bwd(torch.float32, 64, P_CUT, a["vec"], a["ctr"], a["nbr"], a["types"], a["rmax"], a["bw"], a["PQ"], None,
                           torch.zeros(100, 64, device=DEV), a["gvec0"].clone(), nonlin=7, gemm=(a["gouts"], _lib.linear_pack(a["WT"])))


# ---- whole models ------------------------------------------------------------------------------------------------------
def test_c2_model_takes_the_fused_kernel():
    """The c2 architecture on the 3^3 cell: the fp32 model runs the fused kernel and meets the fp64 oracle."""
    oracle, model, d = _pair("c2", 3, "float32")
    _check(oracle, model, d, 1e-4, 1e-4)
    assert model.model._upstream.bwd_path == "fused"


def _four_species_pair(dtype):
    d = systems.make_system("c2", 3)
    g = torch.Generator().manual_seed(11)
    d[D.ATOM_TYPE_KEY] = torch.randint(0, 4, d[D.ATOM_TYPE_KEY].shape, generator=g, dtype=d[D.ATOM_TYPE_KEY].dtype)
    kw = systems.model_kwargs("c2", d[D.EDGE_INDEX_KEY].shape[1] / d[D.POSITIONS_KEY].shape[0], "float64")
    kw.update(type_names=["A", "B", "C", "D"])
    oracle = AllegroOracle(**kw)
    model = AllegroModel(**dict(kw, model_dtype=dtype))
    model.load_state_dict(oracle.state_dict())
    return oracle, model.to(DEV), d


@pytest.mark.parametrize("case", ["fp64", "pq_beyond_smem", "hidden_128"])
def test_model_declines_take_two_launches(case):
    if case == "fp64":
        oracle, model, d = _pair("c2", 3, "float64")
        tol = 1e-9
    elif case == "pq_beyond_smem":
        oracle, model, d = _four_species_pair("float32")
        tol = 1e-4
    else:
        oracle, model, d = _pair("c2", 3, "float32", scalar_embed_mlp_hidden_layers_width=128)
        tol = 1e-4
    _check(oracle, model, d, tol, tol)
    assert model.model._upstream.fold_radial
    assert model.model._upstream.bwd_path == "two_launch"
