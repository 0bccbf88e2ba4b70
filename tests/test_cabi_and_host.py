"""CPU tests: the C-ABI library builds for sm_90a, loads, and exports every symbol that
include/allegro_b200.h declares (no compute calls without a GPU); host-side packing logic."""
import ctypes
import os
import re

import pytest
import torch

from allegro_b200 import _lib, build
from allegro_b200 import data as D
from allegro_b200 import systems
from allegro_b200.model import AllegroModel
from allegro_b200.nn import Contracter
from oracle import nn_ref as R
from oracle import o3_ref
from oracle.model_ref import AllegroOracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    build.build()  # cross-compiles with nvcc; no GPU needed
    return _lib.load()


def test_header_symbols_are_exported(lib):
    hdr = open(os.path.join(ROOT, "include", "allegro_b200.h")).read()
    declared = set(re.findall(r"\b(ab2_\w+)\s*\(", hdr))
    assert len(declared) >= 15
    raw = ctypes.CDLL(_lib.lib_path())
    for sym in declared:
        assert hasattr(raw, sym), f"{sym} declared in the header but not exported"
    assert declared == set(_lib.exported_symbols())
    assert lib.ab2_version() >= 100
    assert lib.ab2_device_ok() in (0, 1)


def test_bad_argument_reports_error(lib):
    # M>0 with null W must fail before any launch (safe without a GPU)
    rc = lib.ab2_linear(1, 4, 8, 8, 0, None, None, None, None, None, 0, None, None, 1, None, None, None, None, 0, None, 0, None)
    assert rc != 0
    assert b"segment" in lib.ab2_last_error()


def test_contracter_tables_equal_oracle_dense_w3j():
    torch.manual_seed(0)
    for irr1, irr2, irro in [("0e+1o+2e", "0e+1o+2e", "0e+1o+2e"), ("0e+1o+2e", "0e+1o+2e", "0e"), ("2o+1e+0e", "0e+0o+1e+1o", "1o+2e")]:
        for coupling in (True, False):
            c = Contracter(irr1, irr2, irro, mul=5, path_channel_coupling=coupling)
            o = R.Contracter(o3_ref.Irreps(irr1), o3_ref.Irreps(irr2), o3_ref.Irreps(irro), mul=5, path_channel_coupling=coupling)
            assert c.w3j.shape == o.w3j.shape and (c.w3j - o.w3j).abs().max() < 1e-6
            o.load_state_dict(c.state_dict())
            # cgw must reproduce the reference's ww3j einsum (_contract.py:218-219)
            ww = torch.einsum(o._weight_w3j_einstr, o.weights, o.w3j).double()
            ijk, _, _ = c.sparse_table()
            cgw = c.cgw(torch.float64, "cpu")
            dense = torch.zeros(5, c.base_dim1, c.base_dim2, c.base_dim_out, dtype=torch.float64)
            for n, (i, j, k) in enumerate(ijk.tolist()):
                dense[:, i, j, k] += cgw[n]
            if o.w3j_is_ij_diagonal:
                full = torch.zeros_like(dense)
                wwu = ww if coupling else ww.unsqueeze(0).expand(5, *ww.shape)
                for i in range(c.base_dim1):
                    full[:, i, i, :] = wwu[:, i, :]
            else:
                full = ww if coupling else ww.unsqueeze(0).expand(5, *ww.shape)
            assert (dense - full).abs().max() < 1e-6


def test_csr_build_and_perm():
    ei = torch.tensor([[2, 0, 1, 0, 2, 2], [0, 1, 2, 2, 1, 0]])
    csr = D.build_csr(ei, 4)
    assert csr.row_ptr.tolist() == [0, 2, 3, 6, 6]
    assert csr.ctr.tolist() == [0, 0, 1, 2, 2, 2]
    assert csr.nbr.tolist() == [1, 2, 2, 0, 1, 0]
    assert csr.perm.tolist() == [1, 3, 2, 0, 4, 5]
    srt = D.build_csr(ei[:, csr.perm], 4)
    assert srt.perm is None and srt.max_degree == 3


def test_model_state_dict_matches_oracle_keys():
    d = systems.make_system("c1")
    kw = systems.model_kwargs("c1", 16.0, "float32")
    m, o = AllegroModel(**kw), AllegroOracle(**kw)
    assert set(m.state_dict().keys()) == set(o.state_dict().keys())
    for k, v in m.state_dict().items():
        assert v.shape == o.state_dict()[k].shape, k
    with pytest.raises(RuntimeError):
        m(d)  # CPU tensors: the hot path refuses, it never falls back


def test_env_perm_is_a_transpose():
    from allegro_b200.nn._pipeline import _env_perm

    U, n_ir = 5, 3
    ref = torch.arange(U * n_ir).view(U, n_ir)  # ref index u*n_ir + r
    assert torch.equal(ref.T.reshape(-1), _env_perm(U, n_ir))


def test_header_is_plain_c_and_links_from_c(tmp_path):
    """The boundary is a C ABI: include/allegro_b200.h must compile as C99 (no C++/torch types) and a C program must
    link against liballegro_b200.so and reach the error plumbing without a GPU (no kernel is launched)."""
    import shutil
    import subprocess

    from allegro_b200._lib import lib_path

    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    inc = os.path.join(root, "include")
    so = lib_path()
    assert os.path.exists(so), "build the extension first (__graft_entry__.build())"
    src = tmp_path / "consumer.c"
    src.write_text(
        '#include <stdio.h>\n#include <string.h>\n#include "allegro_b200.h"\n'
        "int main(void) {\n"
        "  if (ab2_version() <= 0) return 1;\n"
        '  if (ab2_set_option("no_such_option", 1) == 0) return 2;\n'
        '  if (!ab2_last_error() || !strstr(ab2_last_error(), "no_such_option")) return 3;\n'
        '  if (ab2_set_option("tp_fast", 1) != 0) return 4;\n'
        "  /* null-pointer call: argument validation must refuse before any launch */\n"
        "  if (ab2_sh_fwd(AB2_F32, 2, 10, NULL, NULL, NULL) == 0) return 5;\n"
        '  printf("ok %d\\n", ab2_version());\n  return 0;\n}\n'
    )
    exe = tmp_path / "consumer"
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-I", inc, str(src), "-o", str(exe), so, f"-Wl,-rpath,{os.path.dirname(so)}"],
                   check=True, capture_output=True, text=True)
    p = subprocess.run([str(exe)], capture_output=True, text=True)
    assert p.returncode == 0 and p.stdout.startswith("ok"), (p.returncode, p.stdout, p.stderr)
