"""Streaming tensor-product kernels and the other per-centre kernels on ragged neighbour lists, against fp64.

Every case compares ``ab2_tp_fwd`` / ``ab2_tp_bwd`` (through ``_lib``) with an fp64 restatement of the same operation on
the device: the forward is the sum over the table entries, the backward is autograd of that forward, so neither depends
on the hand-derived adjoints.  The reference sees exactly the values the kernel sees (generated in fp64, rounded to the
storage type, converted back).  ``cgw[nnz][U]`` and ``gamma`` are independent random numbers per channel and per entry,
so a swapped channel, entry or channel chunk changes the result.

The CSRs stress the per-centre work split (``cut_centre`` in stream_common.cuh): runs of empty centres (also the first
and the last ones), centres of 1-3 edges that begin inside one 8-edge stage, centres far longer than a stage, one centre
holding more than one CTA's share of the edges, a 5-centre list where most CTAs own no centre, a list with fewer edges
than CTAs, and a c2-sized list.  Which kernel family ran is recorded with torch.profiler and checked against the dispatch
of tp.cu / tp_stream.cu / tp_fast.cu / tp_smem.cu (``_expected_kernels``), so a case cannot pass on another family.
"""
import functools
import os
import re

import pytest
import torch

import kernel_spec
from allegro_b200 import _lib
from tp_dispatch import DEFAULTS, _check_kernels, _expected_for, _families, _from_degrees, _kernels_launched, _ragged_csr
from allegro_b200 import data as D

DEV = "cuda"
SH1, SH2 = "0e+1o", "0e+1o+2e"
L_OF = [0, 1, 1, 1, 2, 2, 2, 2, 2]

# name: (irreps_in1, irreps_in2, irreps_out, implicit V0).  "baked": the structure of Tab9x9x9 / Tab4x4x4
# (tp_tables_generated.cuh), run as straight-line code; the other tables take the general table walk.
SHAPES = {
    "impl9_baked": ("0e+1o+2e", SH2, "0e+1o+2e", True),
    "impl9_t77": ("0e+1o+2e", SH2, "0e+1e+2e", True),
    "expl9_baked": ("0e+1o+2e", SH2, "0e+1o+2e", False),
    "expl9_t63": ("2o+1e+0e", SH2, "0e+1o+2e", False),
    "expl9_t137": ("0e+1e+2e", "0e+1e+2e", "0e+1e+2e", False),
    "last9": ("0e+1o+2e", SH2, "0e", False),
    "impl4_baked": ("0e+1o", SH1, "0e+1o", True),
    "impl4_t10": ("0e+1e", SH1, "0e+1o", True),
    "expl4_baked": ("0e+1o", SH1, "0e+1o", False),
    "expl4_t10": ("0e+1e", SH1, "0e+1o", False),
    # the only tensor product of a one-layer model: implicit V0 straight to the scalar output
    "impl9_last": ("0e+1o+2e", SH2, "0e", True),
    "impl4_last": ("0e+1o", SH1, "0e", True),
}
BAKED = ("impl9_baked", "expl9_baked", "last9", "impl4_baked", "expl4_baked", "impl9_last")
NNZ = {"impl9_baked": 83, "impl9_t77": 77, "expl9_baked": 83, "expl9_t63": 63, "expl9_t137": 137, "last9": 9,
       "impl4_baked": 10, "impl4_t10": 10, "expl4_baked": 10, "expl4_t10": 10, "impl9_last": 9, "impl4_last": 4}


@functools.lru_cache(maxsize=None)
def _table(shape):
    from allegro_b200.nn import Contracter

    a, b, c, _ = SHAPES[shape]
    return Contracter(a, b, c, mul=1).sparse_table()[0].contiguous()


def _dims(shape):
    tab = _table(shape)
    d_in, d_out = int(tab[:, 0].max()) + 1, int(tab[:, 2].max()) + 1
    D_env = 4 if "4" in shape.split("_")[0] else 9
    return d_in, d_out, D_env, SHAPES[shape][3]


# --------------------------------------------------------------------------------------------------------------------
# neighbour lists
# --------------------------------------------------------------------------------------------------------------------
def _csr(kind):
    if kind == "ragged":
        return _ragged_csr(2000, 11, long=True, huge=True)
    if kind == "tiny":  # 5 centres, 40 edges: the CTA cuts at 8, 16, 24 fall inside centre 1, so CTAs own no centre
        return _from_degrees([0, 30, 0, 9, 1], 12)
    if kind == "sparse":  # fewer edges than CTAs: almost every centre is empty
        deg = torch.zeros(600, dtype=torch.int64)
        deg[[7, 8, 300, 301, 302, 590]] = torch.tensor([1, 12, 2, 1, 20, 3])
        return _from_degrees(deg, 13)
    if kind == "c2":  # the benchmark frame's size: 10 976 centres, ~42 edges each
        g = torch.Generator().manual_seed(5)
        return _from_degrees(torch.poisson(torch.full((10976,), 42.0), generator=g).to(torch.int64), 14)
    raise ValueError(kind)


# --------------------------------------------------------------------------------------------------------------------
# fp64 reference of tp_fwd / tp_bwd, any table, any device
# --------------------------------------------------------------------------------------------------------------------
def _tp_sum(tab, cgw, g, V, d_out):
    out = [None] * d_out
    for n, (i, j, k) in enumerate(tab):
        t = cgw[n] * V[:, i] * g[:, j]
        out[k] = t if out[k] is None else out[k] + t
    return torch.stack([o if o is not None else torch.zeros_like(V[:, 0]) for o in out], 1)


def ref_tp(tab, cgw, ctr, gamma, d_out, Vin=None, Y=None, w0=None, gout=None, chunk_elems=1 << 21):
    """Vout[z][k][u] = sum_n cgw[n][u] Vin[z][i][u] gamma[ctr[z]][j][u] over the table entries n = (i, j, k); Vin = Y (x) w0
    (Vin[z][i][u] = Y[z][i] w0[z][l(i)][u]) when ``Vin`` is None.  With ``gout`` also the backward, by autograd of the
    forward: gVin (or gw0 and gY) and ggamma.  Edges are processed in chunks (the sums are linear in each edge's terms)."""
    tab = [tuple(r) for r in tab.tolist()]
    E, N, D, U = ctr.shape[0], gamma.shape[0], gamma.shape[1], gamma.shape[2]
    implicit = Vin is None
    lo = torch.tensor(L_OF[:D], device=gamma.device)
    n_ir = int(lo[-1]) + 1
    res = {"Vout": torch.empty(E, d_out, U, dtype=torch.float64, device=gamma.device)}
    if gout is not None:
        res["ggamma"] = torch.zeros(N, D, U, dtype=torch.float64, device=gamma.device)
        if implicit:
            res["gw0"] = torch.empty(E, n_ir * U, dtype=torch.float64, device=gamma.device)
            res["gY"] = torch.empty(E, D, dtype=torch.float64, device=gamma.device)
        else:
            res["gVin"] = torch.empty(E, Vin.shape[1], U, dtype=torch.float64, device=gamma.device)
    step = max(chunk_elems // (U * D), 1)
    for a in range(0, E, step):
        b = min(a + step, E)
        c = ctr[a:b].long()
        with torch.enable_grad():
            g = gamma[c].detach().requires_grad_(gout is not None)
            if implicit:
                y = Y[a:b].detach().requires_grad_(gout is not None)
                w = w0[a:b, : n_ir * U].detach().requires_grad_(gout is not None)
                V = y.unsqueeze(-1) * w.view(b - a, n_ir, U)[:, lo]
                leaves = (g, y, w)
            else:
                V = Vin[a:b].detach().requires_grad_(gout is not None)
                leaves = (g, V)
            out = _tp_sum(tab, cgw, g, V, d_out)
            res["Vout"][a:b] = out.detach()
            if gout is None:
                continue
            grads = torch.autograd.grad(out, leaves, gout[a:b])
        res["ggamma"].index_add_(0, c, grads[0])
        if implicit:
            res["gY"][a:b] = grads[1]
            res["gw0"][a:b] = grads[2]
        else:
            res["gVin"][a:b] = grads[1]
    return res


def _inputs(shape, dtype, U, csr, seed=0):
    """fp64 values as the kernel sees them (rounded to the storage / accumulation type) on the device."""
    row_ptr, ctr, _ = csr
    N, E = row_ptr.numel() - 1, ctr.numel()
    d_in, d_out, Dd, implicit = _dims(shape)
    acc = _lib.ACC_DTYPE[dtype]
    g = torch.Generator(device=DEV).manual_seed(1000 * seed + U)

    def r(*s, dt, scale=1.0):
        return (torch.randn(*s, generator=g, dtype=torch.float64, device=DEV) * scale).to(dt).double()

    x = {"cgw": r(NNZ[shape], U, dt=acc), "gamma": r(N, Dd, U, dt=acc), "gout": r(E, d_out, U, dt=dtype)}
    if implicit:
        x["Y"] = r(E, Dd, dt=acc)
        x["w0"] = r(E, (int(Dd**0.5)) * U, dt=dtype)
    else:
        x["Vin"] = r(E, d_in, U, dt=dtype)
    x["gY0"] = r(E, Dd, dt=acc) if implicit else None  # gY is accumulated into: a non-zero base
    return x


# --------------------------------------------------------------------------------------------------------------------
# the kernels
# --------------------------------------------------------------------------------------------------------------------
def _set(opts):
    for k, v in opts.items():
        _lib.set_option(k, v)


def _run(shape, dtype, U, csr_dev, x):
    """tp_fwd then tp_bwd; every output prefilled with NaN, gY with the base x["gY0"]."""
    row_ptr, ctr = csr_dev
    N, E = row_ptr.numel() - 1, ctr.numel()
    d_in, d_out, Dd, implicit = _dims(shape)
    acc = _lib.ACC_DTYPE[dtype]
    lmax = 2 if Dd == 9 else 1
    tab = _table(shape).to(DEV)
    f = {k: (v.to(acc if k in ("cgw", "gamma", "Y", "gY0") else dtype) if v is not None else None) for k, v in x.items()}
    nan = float("nan")
    o = {"Vout": torch.full((E, d_out, U), nan, device=DEV, dtype=dtype), "ggamma": torch.full((N, Dd, U), nan, device=DEV, dtype=acc)}
    if implicit:
        o["gw0"] = torch.full((E, f["w0"].shape[1]), nan, device=DEV, dtype=dtype)
        o["gY"] = f["gY0"].clone()
    else:
        o["gVin"] = torch.full((E, d_in, U), nan, device=DEV, dtype=dtype)
    _lib.tp_fwd(dtype, lmax, N, E, U, d_in, d_out, tab, f["cgw"], row_ptr, ctr, f["gamma"], f.get("Vin"), f.get("Y"), f.get("w0"), o["Vout"])
    _lib.tp_bwd(dtype, lmax, N, E, U, d_in, d_out, tab, f["cgw"], row_ptr, ctr, f["gamma"], f.get("Vin"), f.get("Y"), f.get("w0"), f["gout"],
                o.get("gVin"), o.get("gw0"), o.get("gY"), o["ggamma"])
    torch.cuda.synchronize()
    return o


def _expected_kernels(shape, dtype, U, opts):
    """({kernel: template args} of the forward, same of the backward) that ab2_tp_fwd / ab2_tp_bwd launch, from the
    dispatch in tp.cu (streaming kernels first, then tp_fast), tp_stream.cu (ab2_tp_stream, launch_shape),
    tp_fast.cu (launch_fwd / launch_bwd) and tp_smem.cu (tp_variant = 1: MINB = 3; UT = 32 at U = 32).  The template
    arguments are those after the storage and accumulation types."""
    d_in, d_out, D_env, impl = _dims(shape)
    return _expected_for(d_in, d_out, D_env, impl, NNZ[shape], dtype, U, opts)


# --------------------------------------------------------------------------------------------------------------------
# comparison
# --------------------------------------------------------------------------------------------------------------------
def _bars(dtype):
    if dtype == torch.float32:
        return dict(Vout=2e-5, gVin=2e-5, gw0=2e-5, gY=2e-5, ggamma=2e-5)
    return dict(Vout=1e-2, gVin=1e-2, gw0=1e-2, gY=1e-5, ggamma=1e-5)


def compare(got, ref, bars, empty=None, gY0=None):
    """Failures (name, reason) of the kernel outputs ``got`` against the fp64 reference ``ref``: non-finite values, a
    max-abs error above bars[name] * max|ref|, and ggamma rows of empty centres that are not bitwise those of the
    reference (exactly 0).  gY is compared as got - gY0 (the kernel accumulates into the base gY0)."""
    bad = []
    for name, r in ref.items():
        a = got[name].double()
        if name == "gY" and gY0 is not None:
            a = a - gY0.to(a.device, torch.float32).double()
        r = r.to(a.device)
        if not bool(torch.isfinite(a).all()):
            bad.append((name, "non-finite"))
            continue
        err = float((a - r).abs().max()) / max(float(r.abs().max()), 1e-30)
        if not err < bars[name]:
            bad.append((name, f"rel err {err:.3e} >= {bars[name]}"))
        if name == "ggamma" and empty is not None and empty.numel() and not torch.equal(got[name][empty.to(a.device)].double(), r[empty.to(a.device)]):
            bad.append((name, "empty-centre rows differ from 0"))
    return bad


def _rel_errs(got, ref, gY0=None):
    out = {}
    for name, r in ref.items():
        a = got[name].double()
        if name == "gY" and gY0 is not None:
            a = a - gY0.to(a.device, torch.float32).double()
        out[name] = float((a - r.to(a.device)).abs().max()) / max(float(r.abs().max()), 1e-30)
    return out


# --------------------------------------------------------------------------------------------------------------------
# CPU: the reference against the kernel specification, and the sensitivity of the comparison
# --------------------------------------------------------------------------------------------------------------------
def _read_baked_structs():
    path = os.path.join(os.path.dirname(__file__), "..", "allegro_b200", "csrc", "tp_tables_generated.cuh")
    src = open(path).read()
    tabs = {}
    for m in re.finditer(r"struct (\w+) \{(.*?)\n\};", src, re.S):
        arrs = [list(map(int, a.split(","))) for a in re.findall(r"= \{([\d, ]+)\};", m.group(2))]
        if len(arrs) == 3:
            tabs[m.group(1)] = torch.tensor(arrs, dtype=torch.int32).T.contiguous()
    return tabs


def test_table_shapes_are_what_the_kernels_see():
    """The "baked" shapes carry the structure the kernels bake in (tp_tables_generated.cuh), the others do not."""
    baked = _read_baked_structs()
    for shape in SHAPES:
        tab = _table(shape)
        assert tab.shape[0] == NNZ[shape], shape
        d_in, d_out, Dd, _ = _dims(shape)
        ref = {(9, 9): baked["Tab9x9x9"], (4, 4): baked["Tab4x4x4"], (9, 1): baked["Tab9x9x1"]}.get((d_in, d_out))  # no 4 -> 1 struct
        assert (ref is not None and torch.equal(tab, ref)) == (shape in BAKED), shape


def _small_case(shape, seed):
    row_ptr, ctr, _ = _from_degrees([0, 0, 3, 1, 0, 17, 2, 0, 0], seed)
    g = torch.Generator().manual_seed(seed)
    d_in, d_out, Dd, implicit = _dims(shape)
    U, N, E = 5, row_ptr.numel() - 1, ctr.numel()
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)  # noqa: E731
    x = dict(cgw=r(NNZ[shape], U), gamma=r(N, Dd, U), gout=r(E, d_out, U))
    if implicit:
        x.update(Y=r(E, Dd), w0=r(E, int(Dd**0.5) * U))
    else:
        x["Vin"] = r(E, d_in, U)
    return row_ptr, ctr, x, U


@pytest.mark.parametrize("shape", ["impl9_t77", "expl9_t63", "expl9_t137", "impl4_t10", "expl4_t10", "last9", "impl9_last", "impl4_last"])
def test_reference_matches_kernel_spec(shape):
    """The fp64 reference against kernel_spec.tp_fwd / tp_bwd (the executable specification of the C ABI) on a small
    ragged case with empty centres, on the CPU."""
    row_ptr, ctr, x, U = _small_case(shape, 3)
    d_in, d_out, Dd, implicit = _dims(shape)
    N, E, tab = row_ptr.numel() - 1, ctr.numel(), _table(shape)
    ref = ref_tp(tab, x["cgw"], ctr, x["gamma"], d_out, Vin=x.get("Vin"), Y=x.get("Y"), w0=x.get("w0"), gout=x["gout"], chunk_elems=64)
    lmax = 2 if Dd == 9 else 1
    Vout = torch.empty(E, d_out, U, dtype=torch.float64)
    kernel_spec.tp_fwd(None, lmax, N, E, U, d_in, d_out, tab, x["cgw"], row_ptr, ctr, x["gamma"], x.get("Vin"), x.get("Y"), x.get("w0"), Vout)
    spec = {"Vout": Vout, "ggamma": torch.empty(N, Dd, U, dtype=torch.float64)}
    if implicit:
        spec["gw0"], spec["gY"] = torch.empty(E, lmax * U + U, dtype=torch.float64), torch.zeros(E, Dd, dtype=torch.float64)
    else:
        spec["gVin"] = torch.empty(E, d_in, U, dtype=torch.float64)
    kernel_spec.tp_bwd(None, lmax, N, E, U, d_in, d_out, tab, x["cgw"], row_ptr, ctr, x["gamma"], x.get("Vin"), x.get("Y"), x.get("w0"), x["gout"],
                       spec.get("gVin"), spec.get("gw0"), spec.get("gY"), spec["ggamma"])
    assert set(spec) == set(ref)
    for k in ref:
        assert torch.allclose(ref[k], spec[k], rtol=1e-12, atol=1e-12), k


def _corrupt(kind, x, row_ptr):
    """Reference inputs with one small defect, of the kind a kernel bug would leave, at the first centre of 2+ edges."""
    x = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in x.items()}
    c = int(((row_ptr[1:] - row_ptr[:-1]) > 1).nonzero()[0])
    if kind == "swap_gamma_channels":
        x["gamma"][c, :, [0, 1]] = x["gamma"][c, :, [1, 0]]
    elif kind == "drop_last_edge":
        z = int(row_ptr[c + 1]) - 1
        x["gout"][z] = 0
        if "Vin" in x:
            x["Vin"][z] = 0
        else:
            x["w0"][z] = 0
    return x


@pytest.mark.parametrize("shape", ["impl9_t77", "expl9_t63"])
@pytest.mark.parametrize("kind,hit", [("swap_gamma_channels", "Vout"), ("drop_last_edge", "ggamma"), ("empty_centre_ggamma", "ggamma")])
def test_comparison_rejects_small_errors(shape, kind, hit):
    """The comparison the GPU cases use passes a perfect fp32 result and rejects a reference with one small defect:
    two channels of one centre's gamma swapped, the last edge of one centre dropped, one empty centre given a non-zero
    ggamma row (1e-30: far below any value bar, caught by the bitwise empty-row check)."""
    row_ptr, ctr, x, _ = _small_case(shape, 4)
    d_out = _dims(shape)[1]
    tab = _table(shape)

    def ref_of(xx):
        return ref_tp(tab, xx["cgw"], ctr, xx["gamma"], d_out, Vin=xx.get("Vin"), Y=xx.get("Y"), w0=xx.get("w0"), gout=xx["gout"])

    clean = ref_of(x)
    got = {k: v.float() for k, v in clean.items()}  # a kernel that is right up to fp32 rounding
    empty = (row_ptr[1:] == row_ptr[:-1]).nonzero().view(-1)
    bars = _bars(torch.float32)
    assert compare(got, clean, bars, empty) == []
    if kind == "empty_centre_ggamma":
        bad_ref = {k: v.clone() for k, v in clean.items()}
        bad_ref["ggamma"][int(empty[0]), 0, 0] = 1e-30
    else:
        bad_ref = ref_of(_corrupt(kind, x, row_ptr))
    assert hit in {name for name, _ in compare(got, bad_ref, bars, empty)}


# --------------------------------------------------------------------------------------------------------------------
# GPU: the tensor-product matrix
# --------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _csr_dev(kind):
    row_ptr, ctr, _ = _csr(kind)
    return row_ptr.to(DEV), ctr.to(DEV), (row_ptr[1:] == row_ptr[:-1]).nonzero().view(-1).to(DEV)


def _tp_cases():
    cases = []
    for shape in SHAPES:
        for U in (8, 16, 32, 40, 64, 72):
            cases.append((shape, torch.float32, U, "ragged"))
        for U in (8, 32, 40, 64):
            cases.append((shape, torch.bfloat16, U, "ragged"))
    for shape in BAKED:
        for kind in ("tiny", "sparse", "c2"):
            for U in (32, 64):
                for dtype in (torch.float32, torch.bfloat16):
                    cases.append((shape, dtype, U, kind))
    return [pytest.param(*c, id=f"{c[0]}-{str(c[1])[6:]}-U{c[2]}-{c[3]}") for c in cases]


def _stream_outputs(shape, dtype, U, opts):
    """Outputs written by the streaming kernels (every reduction in a fixed order: bitwise reproducible)."""
    fwd, bwd = _expected_kernels(shape, dtype, U, opts)
    implicit = SHAPES[shape][3]
    names = []
    if "tp_stream_kernel" in fwd:
        names.append("Vout")
    if "tp_stream_kernel" in bwd:
        names += ["ggamma"] + (["gw0", "gY"] if implicit else ["gVin"])
    return names


@pytest.mark.gpu
@pytest.mark.parametrize("shape,dtype,U,kind", _tp_cases())
def test_tp_stream_ragged(shape, dtype, U, kind):
    row_ptr, ctr, empty = _csr_dev(kind)
    x = _inputs(shape, dtype, U, (row_ptr, ctr, None))
    d_out = _dims(shape)[1]
    ref = ref_tp(_table(shape).to(DEV), x["cgw"], ctr, x["gamma"], d_out, Vin=x.get("Vin"), Y=x.get("Y"), w0=x.get("w0"), gout=x["gout"])
    bars = _bars(dtype)
    try:
        _set(DEFAULTS)
        got, names = _kernels_launched(lambda: _run(shape, dtype, U, (row_ptr, ctr), x))
        again = _run(shape, dtype, U, (row_ptr, ctr), x)
        _set(dict(tp_stream_cps=1))  # 1 CTA per SM: every CTA boundary moves
        split = _run(shape, dtype, U, (row_ptr, ctr), x)
        # ab2_set_option accepts tp_stream_te, but launch_shape only builds 8-edge stages: the option must stay harmless
        _set(dict(tp_stream_cps=0, tp_stream_te=16))
        te16 = _run(shape, dtype, U, (row_ptr, ctr), x)
    finally:
        _set(DEFAULTS)
    errs = _rel_errs(got, ref, x["gY0"])
    print(f"{shape} {dtype} U={U} {kind}: " + " ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    assert compare(got, ref, bars, empty, x["gY0"]) == []
    assert compare(te16, ref, bars, empty, x["gY0"]) == []
    det = _stream_outputs(shape, dtype, U, DEFAULTS)
    for k in det:
        assert torch.equal(got[k], again[k]), f"{k} differs between two launches"
        # each centre is processed whole by one CTA, in edge order, whatever the grid: the split does not change a bit
        assert torch.equal(got[k], split[k]), f"{k} changes with the work split"
    assert compare(split, ref, bars, empty, x["gY0"]) == []
    if names is None:
        pytest.skip("torch.profiler recorded no CUDA kernel events on this machine: values checked, kernel families not")
    print("  kernels: " + " ".join(_families(names)))
    _check_kernels(names, *_expected_kernels(shape, dtype, U, DEFAULTS))


def _alt_cases():
    cases = []
    for shape in SHAPES:
        for dtype in (torch.float32, torch.bfloat16):
            for U in (32, 64):
                alts = ["tp_stream=0"]
                if shape.startswith("impl9") and dtype == torch.float32 and U == 32:
                    alts += ["tp_stream3=0", "tp_stream3=0,tp_stream_gytile=0"]
                if shape == "last9":
                    alts.append("tp_stream_last=0")
                for a in alts:
                    cases.append(pytest.param(shape, dtype, U, a, id=f"{shape}-{str(dtype)[6:]}-U{U}-{a}"))
    return cases


@pytest.mark.gpu
@pytest.mark.parametrize("shape,dtype,U,alt", _alt_cases())
def test_tp_alternative_builds(shape, dtype, U, alt):
    """The builds the default dispatch does not take at U = 32 and 64 (options of ab2_set_option), on the ragged CSR:
    shared-memory-M / split kernels (tp_stream = 0), the two-warp layer-0 backward with and without the gY tile
    (tp_stream3 = 0, tp_stream_gytile = 0), the 9 -> 1 backward without the streaming kernel (tp_stream_last = 0)."""
    row_ptr, ctr, empty = _csr_dev("ragged")
    x = _inputs(shape, dtype, U, (row_ptr, ctr, None), seed=1)
    ref = ref_tp(_table(shape).to(DEV), x["cgw"], ctr, x["gamma"], _dims(shape)[1], Vin=x.get("Vin"), Y=x.get("Y"), w0=x.get("w0"),
                 gout=x["gout"])
    opts = dict(DEFAULTS)
    opts.update({k: int(v) for k, v in (kv.split("=") for kv in alt.split(","))})
    try:
        _set(opts)
        got, names = _kernels_launched(lambda: _run(shape, dtype, U, (row_ptr, ctr), x))
        again = _run(shape, dtype, U, (row_ptr, ctr), x)
    finally:
        _set(DEFAULTS)
    errs = _rel_errs(got, ref, x["gY0"])
    print(f"{shape} {dtype} U={U} {alt}: " + " ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    assert compare(got, ref, _bars(dtype), empty, x["gY0"]) == []
    for k in _stream_outputs(shape, dtype, U, opts):
        assert torch.equal(got[k], again[k]), f"{k} differs between two launches"
    if names is None:
        pytest.skip("torch.profiler recorded no CUDA kernel events on this machine: values checked, kernel families not")
    print("  kernels: " + " ".join(_families(names)))
    _check_kernels(names, *_expected_kernels(shape, dtype, U, opts))


# --------------------------------------------------------------------------------------------------------------------
# GPU: the other per-centre kernels on the same CSRs
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("rows", ["dense", "strided"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["float32", "bfloat16"])
@pytest.mark.parametrize("U", [32, 40, 64])
@pytest.mark.parametrize("lmax", [1, 2])
def test_env_sum_bwd_ragged(lmax, U, dtype, rows):
    """env_sum / env_bwd against kernel_spec in fp64 on the ragged CSR.  Dense w / gw rows are what the pipeline passes
    (the streaming adjoint, env_stream.cu, takes them at U = 32 and 64); strided rows take the warp-per-centre kernels."""
    row_ptr, ctr, _ = _csr("ragged")
    N, E = row_ptr.numel() - 1, ctr.numel()
    Dd, n_ir = (lmax + 1) ** 2, lmax + 1
    g = torch.Generator().manual_seed(lmax * 100 + U)
    Y = torch.randn(E, Dd, generator=g, dtype=torch.float64).float().double()
    w = torch.randn(E, n_ir * U, generator=g, dtype=torch.float64).to(dtype).double()
    gg = torch.randn(N, Dd, U, generator=g, dtype=torch.float64).float().double()
    gY0 = torch.randn(E, Dd, generator=g, dtype=torch.float64).float()
    sf = 0.3
    gam_ref = kernel_spec.env_sum(dtype, lmax, N, U, row_ptr, Y, w, sf)
    gw_ref, gY_ref = torch.zeros(E, n_ir * U, dtype=torch.float64), torch.zeros(E, Dd, dtype=torch.float64)
    kernel_spec.env_bwd(dtype, lmax, U, ctr, Y, w, gg, sf, gw_ref, gY_ref)

    pad = 0 if rows == "dense" else 3
    wbuf = torch.zeros(E, n_ir * U + 2 * pad, device=DEV, dtype=dtype)
    w_dev = wbuf[:, pad : pad + n_ir * U]
    w_dev.copy_(w.to(dtype))
    gwbuf = torch.full((E, n_ir * U + 2 * pad), float("nan"), device=DEV, dtype=dtype)
    gw_dev = gwbuf[:, pad : pad + n_ir * U]
    gam = torch.full((N, Dd, U), float("nan"), device=DEV)
    rp, ct = row_ptr.to(DEV), ctr.to(DEV)
    _lib.env_sum(dtype, lmax, N, U, rp, Y.float().to(DEV), w_dev, sf, out=gam)
    gY = gY0.to(DEV).clone()
    _lib.env_bwd(dtype, lmax, U, ct, Y.float().to(DEV), w_dev, gg.float().to(DEV), sf, gw_dev, gY, row_ptr=rp)
    torch.cuda.synchronize()

    def rel(a, b):
        return float((a.double().cpu() - b).abs().max()) / float(b.abs().max())

    empty = (row_ptr[1:] == row_ptr[:-1]).nonzero().view(-1)
    assert bool(torch.isfinite(gam).all()) and bool(torch.isfinite(gw_dev).all()) and bool(torch.isfinite(gY).all())
    assert bool((gam[empty.to(DEV)] == 0).all())
    assert rel(gam, gam_ref) < 1e-5
    assert rel(gw_dev, gw_ref) < (1e-5 if dtype == torch.float32 else 1e-2)
    assert rel(gY.double().cpu() - gY0.double(), gY_ref) < 1e-5
    if pad:
        assert bool(torch.isnan(gwbuf[:, :pad]).all()) and bool(torch.isnan(gwbuf[:, -pad:]).all())


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["float64", "float32"])
def test_edge_sum_force_scatter_ragged(dtype):
    """edge_sum / edge_sum_bwd / force_scatter on the ragged CSR with atoms that are nobody's neighbour and ghost rows
    (n_total > N) that receive only the neighbour-side sum; forces bitwise reproducible."""
    N, n_total = 2000, 2300
    g = torch.Generator().manual_seed(8)
    row_ptr, ctr, _ = _ragged_csr(N, 21, long=True, huge=True)
    E = ctr.numel()
    atoms = torch.randperm(n_total, generator=g)
    pool = atoms[: n_total - 400]  # 400 atoms, owned and ghost, are nobody's neighbour
    nbr = pool[torch.randint(0, pool.numel(), (E,), generator=g)].to(torch.int32)
    lonely = atoms[n_total - 400 :]
    assert bool((lonely < N).any()) and bool((lonely >= N).any())
    csr = D.EdgeCSR(N, ctr.to(DEV), nbr.to(DEV), row_ptr.to(DEV), None, int((row_ptr[1:] - row_ptr[:-1]).max()))
    tol = 1e-12 if dtype == torch.float64 else 2e-5
    empty = (row_ptr[1:] == row_ptr[:-1]).nonzero().view(-1)

    Ez = torch.randn(E, generator=g, dtype=torch.float64).to(dtype).double()
    Ei = _lib.edge_sum(Ez.to(DEV, dtype), row_ptr.to(DEV), 0.25)
    Ei_ref = torch.zeros(N, dtype=torch.float64).index_add_(0, ctr.long(), 0.25 * Ez)
    assert float((Ei.double().cpu() - Ei_ref).abs().max()) < tol * float(Ei_ref.abs().max())
    assert bool((Ei.cpu()[empty] == 0).all())

    gEi = torch.randn(N, generator=g, dtype=torch.float64).to(dtype).double()
    gEz = _lib.edge_sum_bwd(gEi.to(DEV, dtype), ctr.to(DEV), 0.25)
    assert float((gEz.double().cpu() - 0.25 * gEi[ctr.long()]).abs().max()) <= tol * float(gEi.abs().max())

    gv = torch.randn(E, 3, generator=g, dtype=torch.float64).to(dtype).double()
    F = _lib.force_scatter(gv.to(DEV, dtype), csr, n_total)
    assert F.shape == (n_total, 3)
    assert torch.equal(F, _lib.force_scatter(gv.to(DEV, dtype), csr, n_total))
    F_ref = torch.zeros(n_total, 3, dtype=torch.float64).index_add_(0, ctr.long(), gv).index_add_(0, nbr.long(), -gv)
    assert float((F.double().cpu() - F_ref).abs().max()) < 10 * tol * float(F_ref.abs().max())
    # rows with neither side (empty owned centres that are nobody's neighbour) are exactly 0
    none = [a for a in lonely.tolist() if a >= N or int(row_ptr[a + 1] - row_ptr[a]) == 0]
    assert bool((F.cpu()[none] == 0).all())


# --------------------------------------------------------------------------------------------------------------------
# GPU: whole models on the stored-feature kernels at c3 widths
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_c3_widths_stored_v_fp32(monkeypatch):
    """c3 widths (S = 128, U = 64: the two-chunk UT = 64 builds) on the 6^3 reduced cell, with the composed two-layer
    path declined so that the model runs on the stored-feature tensor-product kernels."""
    from allegro_b200 import _lib
    from test_gpu_model import _check, _pair

    monkeypatch.setattr(_lib, "tp_chain_plan", lambda *a: None)
    oracle, model, d = _pair("c3", 6, "float32")
    core = model.model.core()
    assert core.U == 64 and core.chain is None
    ee, ef = _check(oracle, model, d, 1e-4, 1e-4)
    print(f"c3 widths fp32 stored V: E {ee:.2e} F {ef:.2e}")


@pytest.mark.gpu
def test_c3_widths_bf16():
    """The same cell in bf16 storage (the composed path is fp32-only), at the bars of the c2 bf16 model test."""
    from test_gpu_model import _check, _pair

    oracle, model, d = _pair("c3", 6, "bfloat16")
    core = model.model.core()
    assert core.U == 64 and core.chain is None
    ee, ef = _check(oracle, model, d, 2e-2, 5e-2)
    print(f"c3 widths bf16: E {ee:.2e} F {ef:.2e}")


# --------------------------------------------------------------------------------------------------------------------
# GPU: which kernels serve the l_max 4 tables (values: test_gpu_kernels.test_tp_lmax4_ragged_generic and the explicit /
# implicit grids there)
# --------------------------------------------------------------------------------------------------------------------
LMAX4_TABLES = {"25to25": (2, 0), "25to49": (3, 0), "49to25": (3, 1), "25to1": (3, 2)}  # (L, layer) of an l_max 4 model
LMAX4_DTYPES = {"float64": torch.float64, "float32": torch.float32, "bfloat16": torch.bfloat16}


def _lmax4_trace(table, dtype):
    """(d_in, d_out, D, implicit, nnz, names of the kernels ab2_tp_fwd + ab2_tp_bwd launch under the default options) of one
    l_max 4 table on a small ragged CSR with empty centres."""
    from test_gpu_kernels import _tp_case

    L, layer = LMAX4_TABLES[table]
    lmax, U, N = 4, 32, 9
    _, b = _tp_case(lmax, layer, L, U, True, dtype)
    implicit = layer == 0
    d_in, d_out, Dd = b.base_dim1, b.base_dim_out, (lmax + 1) ** 2
    ijk, _, _ = b.sparse_table()
    acc = _lib.ACC_DTYPE[dtype]
    tab, cgw = ijk.to(DEV), b.cgw(acc, DEV)
    g = torch.Generator().manual_seed(L * 10 + layer)
    deg = torch.tensor([0, 5, 1, 0, 12, 3, 0, 7, 0])
    ctr = torch.repeat_interleave(torch.arange(N), deg)
    E = int(ctr.numel())
    csr = D.build_csr(torch.stack([ctr, torch.randint(0, N, (E,), generator=g)]).to(DEV), N)
    dd = dict(dtype=torch.float64, generator=g)
    yw = (torch.randn(E, Dd, **dd).to(DEV, acc), torch.randn(E, (lmax + 1) * U, **dd).to(DEV, dtype)) if implicit else (None, None)
    Vin = None if implicit else torch.randn(E, d_in, U, **dd).to(DEV, dtype)
    gam, gout = torch.randn(N, Dd, U, **dd).to(DEV, acc), torch.randn(E, d_out, U, **dd).to(DEV, dtype)

    def run():
        Vout = torch.empty(E, d_out, U, device=DEV, dtype=dtype)
        gVin = None if implicit else torch.empty(E, d_in, U, device=DEV, dtype=dtype)
        gw0 = torch.empty(E, (lmax + 1) * U, device=DEV, dtype=dtype) if implicit else None
        gY = torch.zeros(E, Dd, device=DEV, dtype=acc) if implicit else None
        ggam = torch.empty(N, Dd, U, device=DEV, dtype=acc)
        _lib.tp_fwd(dtype, lmax, N, E, U, d_in, d_out, tab, cgw, csr.row_ptr, csr.ctr, gam, Vin, *yw, Vout)
        _lib.tp_bwd(dtype, lmax, N, E, U, d_in, d_out, tab, cgw, csr.row_ptr, csr.ctr, gam, Vin, *yw, gout, gVin, gw0, gY, ggam)
        torch.cuda.synchronize()
        return bool(torch.isfinite(Vout).all())

    _set(DEFAULTS)
    finite, names = _kernels_launched(run)
    assert finite
    return d_in, d_out, Dd, implicit, int(tab.shape[0]), names


_LMAX4_FRESH_PROCESS = r"""
import json, sys
sys.path[:0] = [{root!r}, {tests!r}]
import test_gpu_tp_ragged as T
out = {{}}
for table in T.LMAX4_TABLES:
    for dname, dtype in T.LMAX4_DTYPES.items():
        out[table + "-" + dname] = T._lmax4_trace(table, dtype)
print("TRACES " + json.dumps(out))
"""


@pytest.fixture(scope="module")
def lmax4_traces():
    """The traces of every l_max 4 table and dtype, taken in a fresh process: in one long pytest process, traces taken after
    many earlier profiler sessions have lacked kernel records (the forward kernel's, while the values were right), so these
    tables are traced where no earlier session runs and add no sessions to the process of the other trace checks."""
    import json
    import subprocess
    import sys

    here = os.path.dirname(os.path.abspath(__file__))
    code = _LMAX4_FRESH_PROCESS.format(root=os.path.dirname(here), tests=here)
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code], capture_output=True, text=True,
                       timeout=900)
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("TRACES ")]
    assert r.returncode == 0 and line, r.stdout[-2000:] + r.stderr[-4000:]
    return json.loads(line[-1][len("TRACES "):])


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", list(LMAX4_DTYPES))
@pytest.mark.parametrize("table", list(LMAX4_TABLES))
def test_lmax4_tables_run_the_generic_kernels(table, dtype, lmax4_traces):
    """No fast family takes an l_max 4 table (25 -> 25, 25 -> 49, 49 -> 25, 25 -> 1): under the default options ab2_tp_fwd /
    ab2_tp_bwd run tp_fwd_generic_kernel / tp_bwd_generic_kernel and no other tensor-product kernel.  A later fast kernel
    for these tables changes this expectation and comes with its own test."""
    d_in, d_out, Dd, implicit, nnz, names = lmax4_traces[f"{table}-{dtype}"]
    if names is None:
        pytest.skip("torch.profiler recorded no CUDA kernel events on this machine")
    print(f"  l_max 4 {d_in} -> {d_out} ({nnz} entries) {dtype}: " + " ".join(_families(names)))
    _check_kernels(names, *_expected_for(d_in, d_out, Dd, implicit, nnz, LMAX4_DTYPES[dtype], 32, DEFAULTS))
