"""The C-ABI library: exports every symbol include/dab200.h declares, and fails loudly without a GPU."""
import ctypes
import os
import re

import numpy as np
import pytest

from tests.common import ROOT, setup

LIB = os.path.join(ROOT, "dafoam_b200", "libdab200.so")


def declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "dab200.h")).read()
    return sorted(set(re.findall(r"\b(dab_[a-z0-9_]+)\s*\(", hdr)))


@pytest.mark.skipif(not os.path.exists(LIB), reason="libdab200.so not built (run __graft_entry__.build())")
def test_library_exports_every_declared_symbol():
    L = ctypes.CDLL(LIB)
    syms = declared_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(L, s), "missing symbol " + s
    L.dab_version.restype = ctypes.c_char_p
    assert b"sm_90a" in L.dab_version()


@pytest.mark.skipif(not os.path.exists(LIB), reason="libdab200.so not built")
def test_no_cpu_fallback_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible")
    from dafoam_b200.pyDASolvers import DAB200Error
    with pytest.raises(DAB200Error, match="requires a CUDA device"):
        setup("channel", True, nk=1, with_oracle=False)


def test_missing_library_is_an_error():
    from dafoam_b200.pyDASolvers import DAB200Error, load_library
    with pytest.raises(DAB200Error, match="no CPU fallback"):
        load_library("/nonexistent/libdab200.so")


def test_argument_errors_mirror_the_reference():
    from tests.common import HOSTSIM
    mesh, bcs, orc, sol, W, _ = setup("channel", False, nk=1, lib_path=HOSTSIM)
    with pytest.raises(AssertionError, match="invalid"):
        sol.updateOFFields(np.zeros(3))
    from dafoam_b200.pyDASolvers import DAB200Error
    with pytest.raises(DAB200Error, match="not supported"):
        sol.calcJacTVecProduct("x", "regressionPar", np.zeros(1), "R", "residual", np.zeros(orc.ndof), np.zeros(1)) if False else \
            sol._raise(sol._L.dab_calc_jac_t_vec_product(sol._h, b"x", b"regressionPar", None, b"R", b"residual",
                                                         W.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                                         W.ctypes.data_as(ctypes.POINTER(ctypes.c_double))))
    with pytest.raises(DAB200Error, match="is not defined"):
        sol.calcFunction("CL")


def test_output_and_statistics_helpers(capsys):
    """calcOutput / calcPrimalResidualStatistics / BC refresh no-ops of the reference's pyDASolvers API."""
    from dafoam_b200.pyDASolvers import DAB200Error
    from tests.common import HOSTSIM
    fn = {"CD": {"type": "force", "source": "patchToFace", "patches": ["wing"], "directionMode": "fixedDirection",
                 "direction": [1.0, 0.0, 0.0], "scale": 0.02}}
    mesh, bcs, orc, sol, W, _ = setup("naca", True, nk=1, lib_path=HOSTSIM, extra_options=dict(function=fn))
    sol.updateOFFields(W)
    sol.updateStateBoundaryConditions()
    sol.updateBoundaryConditions("U", "vector")
    with pytest.raises(DAB200Error):
        sol.updateBoundaryConditions("U", "tensor")
    R = np.zeros(orc.ndof)
    sol.calcOutput("R", "residual", R)
    R2 = np.zeros(orc.ndof)
    sol.getResiduals(R2)
    assert np.array_equal(R, R2)
    st = sol.calcPrimalResidualStatistics("print")
    txt = capsys.readouterr().out
    assert "U Residual Norm2: (" in txt and "Total Residual Norm2" in txt
    assert abs(st["total"] - np.linalg.norm(R)) <= 1e-12 * np.linalg.norm(R)
    nC = mesh.n_cells
    assert np.allclose(st["nuTilda"]["max"], np.abs(R[4 * nC:5 * nC]).max())
    with pytest.raises(DAB200Error):
        sol.calcPrimalResidualStatistics("dump")
    name = list(sol._options["function"].keys())[0]
    v = np.zeros(1)
    sol.calcOutput(name, "function", v)
    assert v[0] == sol.calcFunction(name)


def test_new_entry_points_reject_bad_arguments():
    """NULL handles / pointers and impossible requests of the file, mesh-check and solver entry points return an error code with a
    message (never a crash), through the raw C ABI."""
    from dafoam_b200.pyDASolvers import DAB200Error
    from tests.common import HOSTSIM
    mesh, bcs, orc, sol, W, _ = setup("channel", True, nk=1, lib_path=HOSTSIM)
    L, h = sol._L, sol._h
    dp = ctypes.POINTER(ctypes.c_double)
    ok = ctypes.c_int(0)
    assert L.dab_check_mesh(None, ctypes.c_double(70), ctypes.c_double(4), ctypes.c_double(1000), 0, ctypes.byref(ok), None) != 0
    assert L.dab_check_mesh(h, ctypes.c_double(70), ctypes.c_double(4), ctypes.c_double(1000), 0, None, None) != 0
    assert L.dab_check_mesh(h, ctypes.c_double(70), ctypes.c_double(4), ctypes.c_double(1000), 0, ctypes.byref(ok), None) == 0 and ok.value == 1
    assert L.dab_read_state_vars(h, ctypes.c_double(12345.0)) != 0 and b"does not exist" in L.dab_last_error()
    assert L.dab_read_mesh_points(h, ctypes.c_double(12345.0)) != 0
    assert L.dab_write_mesh_points(h, None, None) != 0
    assert L.dab_write_sens_map_field(h, b"s", W.ctypes.data_as(dp), b"tensor", ctypes.c_double(1.0)) != 0
    assert L.dab_write_sens_map_surface(h, b"s", None, None, 3, ctypes.c_double(1.0), None) != 0
    assert L.dab_run_fp_adj(h, None, None, None, None) != 0
    with pytest.raises(DAB200Error, match="old-time levels"):
        sol.readStateVars(0.0, 1)
    with pytest.raises(DAB200Error):
        sol.getOFFieldGlobal("p", "vector", np.zeros(3))
    with pytest.raises(DAB200Error, match="not found"):
        sol.getdFScaling("CL")
    # a surface map with no design points is refused
    with pytest.raises(DAB200Error, match="empty surface"):
        sol.writeSensMapSurface("s", np.zeros(0), np.zeros(0), 0, 1.0)
