"""Which tensor-product kernels ``ab2_tp_fwd`` / ``ab2_tp_bwd`` launch, and the ragged neighbour lists the tests run them on.

``_expected_for`` restates the dispatch of tp.cu in its order: the streaming kernels of tp_stream.cu (``ab2_tp_stream``,
``launch_shape``) first, then the tp_fast / tp_smem builds (``ab2_tp_fast_supported``, tp_fast.cu ``launch_fwd`` /
``launch_bwd``, tp_smem.cu at tp_variant = 1: MINB = 3, UT = 32 at U = 32), then the shape-generic kernels.
``_kernels_launched`` records with torch.profiler which kernels ran, ``_check_kernels`` holds them to a prediction.
Used by test_gpu_tp_ragged.py (the kernels through ``_lib``) and test_gpu_operator.py (the same kernels behind
``allegro_b200.nn.Contracter``)."""
import re

import torch

# (d_in, d_out, D) that tp_fast.cu (AB2_FAST_SHAPES) and tp_smem.cu (AB2_SMEM_SHAPES) are built for
FAST_SHAPES = {(4, 4, 4), (4, 1, 4), (9, 9, 9), (9, 1, 9), (16, 1, 16), (7, 4, 4), (4, 7, 4), (7, 7, 4), (7, 1, 4)}
DEFAULTS = dict(tp_fast=1, tp_stream=1, tp_stream3=1, tp_stream_gytile=1, tp_stream_last=1, tp_stream_te=0, tp_stream_cps=0)
STREAM_MAX_NNZ = 256  # MAX_NNZ of tp_stream.cu

FAMILIES = ("tp_stream_kernel", "tp_stream_gyt_kernel", "tp_bwd3_kernel", "tp_smem_kernel", "tp_fwd_fast_kernel", "tp_bwd_fast_kernel",
            "tp_bwd_gm_split_kernel", "tp_fwd_generic_kernel", "tp_bwd_generic_kernel")


# --------------------------------------------------------------------------------------------------------------------
# neighbour lists
# --------------------------------------------------------------------------------------------------------------------
def _from_degrees(deg, seed, n_nbr=None):
    g = torch.Generator().manual_seed(seed)
    deg = torch.as_tensor(deg, dtype=torch.int64)
    N = deg.numel()
    row_ptr = torch.zeros(N + 1, dtype=torch.int64)
    row_ptr[1:] = torch.cumsum(deg, 0)
    ctr = torch.repeat_interleave(torch.arange(N), deg)
    nbr = torch.randint(0, n_nbr or N, (ctr.numel(),), generator=g)
    return row_ptr.to(torch.int32), ctr.to(torch.int32), nbr.to(torch.int32)


def _ragged_csr(N, seed, long=True, huge=False):
    """Degrees with runs of empty centres (the first 5 and the last 7 among them), ~30 % of the centres with 1-3 edges,
    the rest with 4-20, some of 60-300 edges (``long``) and optionally one centre of ~E/100 edges (``huge``: more than
    one CTA's share at the default grid of a few CTAs per SM)."""
    g = torch.Generator().manual_seed(seed)
    deg = torch.randint(4, 21, (N,), generator=g)
    short = torch.rand(N, generator=g) < 0.3
    deg[short] = torch.randint(1, 4, (int(short.sum()),), generator=g)
    for s in torch.randint(0, N, (max(N // 60, 1),), generator=g).tolist():
        deg[s : s + int(torch.randint(1, 9, (1,), generator=g))] = 0
    if long:
        idx = torch.randperm(N, generator=g)[: max(N // 40, 1)]
        deg[idx] = torch.randint(60, 301, (idx.numel(),), generator=g)
    deg[:5] = 0
    deg[-7:] = 0
    if huge:
        deg[N // 2] = int(deg.sum()) // 99
    return _from_degrees(deg, seed + 1)


# --------------------------------------------------------------------------------------------------------------------
# the dispatch
# --------------------------------------------------------------------------------------------------------------------
def _stream_build(U, dtype=torch.float32):
    """(NCH, TE, NS, UT) of launch_shape in tp_stream.cu, None where ab2_tp_stream or launch_shape declines the width:
    rows of U elements must be whole 16-byte multiples (bulk copies), and U <= 64."""
    esz = 4 if dtype == torch.float32 else 2
    if (U * esz) % 16 or (U * 4) % 16:
        return None
    if U == 32:
        return (1, 8, 3, 32)
    if U < 32:
        return (1, 8, 3, 0)
    if U == 64:
        return (2, 8, 2, 64)
    if U < 64:
        return (2, 8, 2, 0)
    return None


def _b(v):
    return "true" if v else "false"


def _stream_takes(mode, d_in, d_out, D_env, impl, nnz, dtype, opts):
    """The shape conditions of ab2_tp_stream (mode 0 forward, 1 backward): fp32 / bf16, at most MAX_NNZ entries, and
    d_in == d_out in {4, 9} with any D for explicit input features (implicit V0 needs D == d_in), or the explicit 9 -> 1
    backward at D = 9."""
    if not (opts["tp_fast"] and opts["tp_stream"]) or dtype not in (torch.float32, torch.bfloat16) or not 0 < nnz <= STREAM_MAX_NNZ:
        return False
    if mode == 1 and opts["tp_stream_last"] and not impl and (d_in, d_out, D_env) == (9, 1, 9):
        return True
    return d_in == d_out and d_in in (4, 9) and (not impl or D_env == d_in)


def _expected_for(d_in, d_out, D_env, impl, nnz, dtype, U, opts):
    """({kernel: template args} of the forward, same of the backward) that ab2_tp_fwd / ab2_tp_bwd launch for a table
    d_in -> d_out with D_env spherical-harmonic components, implicit V0 or not, nnz entries.  The template arguments are
    those after the storage and accumulation types; the generic kernels have none: ()."""
    build = _stream_build(U, dtype)
    fast = dtype in (torch.float32, torch.bfloat16) and opts["tp_fast"] and (d_in, d_out, D_env) in FAST_SHAPES and (not impl or d_in == D_env)
    ut = 32 if U == 32 else 0

    if build and _stream_takes(0, d_in, d_out, D_env, impl, nnz, dtype, opts):
        fwd = {"tp_stream_kernel": (d_in, d_out, _b(impl), 0) + build}
    elif fast:
        fwd = {"tp_smem_kernel": (d_in, d_out, _b(impl), 0, 3, ut)}
    else:
        fwd = {"tp_fwd_generic_kernel": ()}

    if build and _stream_takes(1, d_in, d_out, D_env, impl, nnz, dtype, opts):
        if d_out == 1:
            bwd = {"tp_stream_kernel": (9, 1, "false", 1) + build}
        else:
            args = (d_in, d_out, _b(impl), 1) + build
            bwd = {"tp_stream_kernel": args}
            if impl and d_in == 9 and dtype == torch.float32 and U == 32:
                if opts["tp_stream3"] and nnz == 83:
                    bwd["tp_bwd3_kernel"] = ("false", 1)  # then the two-warp kernel, standing down on the baked table
                elif opts["tp_stream_gytile"]:
                    bwd["tp_stream_gyt_kernel"] = args  # works on the baked table, the plain build behind it otherwise
    elif fast and d_in * d_out >= 49:
        bwd = {"tp_smem_kernel": (d_in, d_out, _b(impl), 1, 3, ut), "tp_bwd_gm_split_kernel": (d_in, d_out, D_env, _b(impl), 3)}
    elif fast:
        bwd = {"tp_bwd_fast_kernel": (d_in, d_out, D_env, _b(impl), "false")}
    else:
        bwd = {"tp_bwd_generic_kernel": ()}
    return fwd, bwd


# --------------------------------------------------------------------------------------------------------------------
# what ran
# --------------------------------------------------------------------------------------------------------------------
def _template_args(name, family):
    m = re.search(r"\b" + family + "<", name)
    if not m:
        return None
    depth, i = 1, m.end()
    while depth and i < len(name):
        depth += {"<": 1, ">": -1}.get(name[i], 0)
        i += 1
    return [a.strip() for a in name[m.end() : i - 1].split(",")]


def _kernels_launched(fn, runs=5):
    """(result of the first fn(), sorted names of the CUDA kernels fn launches) from torch.profiler's CUDA activity;
    names is None when the profiler sees no kernel at all.

    One trace is not complete evidence: now and then it is empty, or it lacks the records of some kernels that ran (in a
    long pytest process, a forward or backward tensor-product kernel was missing while the values were right, in two
    consecutive traces).  So fn runs under the profiler ``runs`` times, and names is the union of what the traces saw:
    it holds only kernels that ran, so a family that was not launched can never appear in it, and a kernel is missed
    only if every trace drops it."""
    from torch.profiler import ProfilerActivity, profile

    out, union = None, set()
    for _ in range(runs):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            res = fn()
        out = res if out is None else out
        names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        union |= {n for n in names if not n.startswith(("Memset", "Memcpy"))}
    return out, (sorted(union) if union else None)


def _families(names):
    return sorted({f"{f}<{', '.join(_template_args(n, f)[2:] if f != 'tp_bwd3_kernel' else _template_args(n, f))}>"
                   for n in names for f in FAMILIES if _template_args(n, f) is not None})


def _check_kernels(names, fwd, bwd):
    """Every expected family appears with its template arguments, and no other tensor-product family does."""
    seen = {f for n in names for f in FAMILIES if _template_args(n, f) is not None}
    assert seen == set(fwd) | set(bwd), (sorted(seen), fwd, bwd, names)
    for want in (fwd, bwd):
        for fam, args in want.items():
            got = [_template_args(n, fam) for n in names if _template_args(n, fam) is not None]
            exp = [str(a) for a in args]
            assert any(g[len(g) - len(exp):] == exp for g in got), (fam, exp, got)  # exp may be empty (generic kernels)
