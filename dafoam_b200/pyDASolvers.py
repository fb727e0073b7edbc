"""pyDASolvers -- the Python face of the drop-in boundary.

Mirrors the reference's Cython class `pyDASolvers` (reference src/pyDASolvers/pyDASolvers.pyx:117-483):
same method names, same argument meaning (caller-allocated C-contiguous float64 numpy arrays,
size-asserted), same soft-failure convention (integer returns for solvePrimal/solveLinearEqn, hard
errors raise).  Implemented as a thin ctypes binding of the C ABI in include/dab200.h; there is no CPU
fallback: if libdab200.so (CUDA, sm_90a) is missing or no GPU is visible, construction raises.

petsc4py is not available in this environment, so the PETSc handle arguments of the reference
(`Mat`, `KSP`, `Vec`) are replaced by tiny handle classes defined here (`Mat`, `KSP`) and by plain
numpy arrays for vectors; the call sequence of `DAFoamSolver.solve_linear`
(reference dafoam/mphys/mphys_dafoam.py:433-574) is preserved.
"""
from __future__ import annotations

import ctypes as C
import json
import os
import time
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIBS = {}


class DAB200Error(RuntimeError):
    pass


class KspStats(C.Structure):
    _fields_ = [("iterations", C.c_int32), ("converged_reason", C.c_int32), ("initial_residual", C.c_double),
                ("final_residual", C.c_double), ("solve_seconds", C.c_double), ("pc_setup_seconds", C.c_double),
                ("n_matvec", C.c_int32), ("pc_assemblies", C.c_int32)]


class PrimalStats(C.Structure):
    _fields_ = [("iterations", C.c_int32), ("converged", C.c_int32), ("p_iterations", C.c_int32), ("reserved", C.c_int32),
                ("max_residual", C.c_double), ("res_u", C.c_double * 3), ("res_p", C.c_double), ("res_nutilda", C.c_double),
                ("seconds", C.c_double)]


def load_library(path=None):
    """Load libdab200.so.  `path` is only used by the test-suite to load the host-simulation build."""
    path = path or os.path.join(_HERE, "libdab200.so")
    if path in _LIBS:
        return _LIBS[path]
    if not os.path.exists(path):
        raise DAB200Error("%s not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(there is no CPU fallback)" % path)
    L = C.CDLL(path)
    L.dab_last_error.restype = C.c_char_p
    L.dab_version.restype = C.c_char_p
    _LIBS[path] = L
    return L


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _check_array(a, n, what):
    assert isinstance(a, np.ndarray) and a.dtype == np.float64 and a.flags["C_CONTIGUOUS"], "%s must be a C-contiguous float64 array" % what
    assert len(a) == n, "invalid %s array size!" % what


EXCHANGE_CB = C.CFUNCTYPE(None, C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.POINTER(C.c_double)), C.POINTER(C.c_int),
                          C.POINTER(C.POINTER(C.c_double)), C.POINTER(C.c_int))
ALLREDUCE_CB = C.CFUNCTYPE(None, C.c_void_p, C.POINTER(C.c_double), C.c_int)
_CB_KEEP = []


def nccl_unique_id(lib_path=None):
    """128-byte NCCL unique id (rank 0 creates it, the caller broadcasts it, every rank passes it to pyDASolvers)."""
    L = load_library(lib_path)
    buf = C.create_string_buffer(128)
    if L.dab_nccl_unique_id(buf) != 0:
        raise DAB200Error(L.dab_last_error().decode())
    return buf.raw


def set_comm_callbacks(exchange, allreduce, lib_path):
    """TEST BUILD ONLY: route halo exchanges / all-reduces of the next solver through Python callables
    exchange(peers, send_arrays, recv_arrays) and allreduce(array) (numpy views of the library's buffers)."""
    L = load_library(lib_path)

    def _ex(ctx, n, peers, sb, sc, rb, rc):
        ps = [peers[i] for i in range(n)]
        sends = [np.ctypeslib.as_array(sb[i], shape=(sc[i],)) if sc[i] > 0 else np.zeros(0) for i in range(n)]
        recvs = [np.ctypeslib.as_array(rb[i], shape=(rc[i],)) if rc[i] > 0 else np.zeros(0) for i in range(n)]
        exchange(ps, sends, recvs)

    def _ar(ctx, buf, n):
        allreduce(np.ctypeslib.as_array(buf, shape=(n,)))

    cbs = (EXCHANGE_CB(_ex), ALLREDUCE_CB(_ar))
    _CB_KEEP.append(cbs)
    if L.dab_set_comm_callbacks(cbs[0], cbs[1], None) != 0:
        raise DAB200Error(L.dab_last_error().decode())


class Mat:
    """Stand-in for the PETSc Mat handle of the reference's calcdRdWT(isPC, dRdWT) / calcPCMatWithFvMatrix(PCMat, turbOnly)."""

    def __init__(self):
        self.assembled = False
        self.rows = self.cols = self.vals = None  # COO triplets inserted by calcPCMatWithFvMatrix (INSERT_VALUES)

    def zeroEntries(self):
        self.rows = self.cols = self.vals = None

    def norm(self):
        """Frobenius norm (petsc4py Mat.norm() default, as the reference's unit test reads it)."""
        return 0.0 if self.vals is None else float(np.sqrt(np.sum(self.vals * self.vals)))

    def toDense(self, n):
        a = np.zeros((n, n))
        if self.vals is not None:
            a[self.rows, self.cols] = self.vals
        return a


class KSP:
    """Stand-in for the PETSc KSP handle (createMLRKSPMatrixFree / solveLinearEqn)."""

    def __init__(self):
        self.ready = False
        self.stats = None


class pyDASolvers:
    def __init__(self, argsAll, pyOptions, caseDir=".", device=0, rank=0, nRanks=1, ncclUniqueId=None, _lib_path=None):
        """argsAll: e.g. "DASimpleFoam -python"; pyOptions: the DAOPTION dict (reference dafoam/pyDAFoam.py:39-662).
        caseDir replaces the reference's implicit os.getcwd() case directory."""
        self._L = load_library(_lib_path)
        self._h = C.c_void_p()
        if isinstance(argsAll, bytes):
            argsAll = argsAll.decode()
        self._options = dict(pyOptions or {})
        self._solverName = argsAll.split()[0] if argsAll.split() else "DASimpleFoam"
        self._caseDir, self._rank, self._nRanks = os.path.abspath(caseDir), rank, nRanks
        uid = None if ncclUniqueId is None else C.c_char_p(bytes(ncclUniqueId))
        rc = self._L.dab_create(os.path.abspath(caseDir).encode(), argsAll.encode(), json.dumps(self._options).encode(),
                                C.c_int(device), C.c_int(rank), C.c_int(nRanks), uid, C.byref(self._h))
        self._raise(rc)
        self._initialised = False
        self._t0Clock, self._t0Cpu = time.time(), time.process_time()

    # ---- plumbing
    def _raise(self, rc):
        if rc != 0:
            raise DAB200Error(self._L.dab_last_error().decode())

    def _geti(self, fn):
        v = C.c_int64()
        self._raise(fn(self._h, C.byref(v)))
        return int(v.value)

    def __del__(self):
        try:
            if self._h:
                self._L.dab_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass

    # ---- the reference's methods (pyDASolvers.pyx)
    def initSolver(self):
        self._initialised = True

    def getNLocalAdjointStates(self):
        return self._geti(self._L.dab_n_local_adjoint_states)

    def getNLocalCells(self):
        return self._geti(self._L.dab_n_local_cells)

    def getNGlobalCells(self):
        return self._geti(self._L.dab_n_global_cells)

    def getNLocalPoints(self):
        return self._geti(self._L.dab_n_local_points)

    def getVolCoordEvaluations(self):
        """residual evaluations of one volCoord product (colouring of the first product; the same on every rank)"""
        return self._geti(self._L.dab_volcoord_evaluations)

    def getNLocalFaces(self):
        return self._geti(self._L.dab_n_local_faces)

    def getNLocalInternalFaces(self):
        return self._geti(self._L.dab_n_local_internal_faces)

    def getLocalToGlobal(self, what):
        """what: "cells" -> global cell ids, "faces" -> global face ids, "faceOwned" -> 0/1 ownership of the phi DOF."""
        code = {"cells": 0, "faces": 1, "faceOwned": 2}[what]
        n = self.getNLocalCells() if code == 0 else self.getNLocalFaces()
        out = np.zeros(n, dtype=np.int64)
        self._raise(self._L.dab_get_local_to_global(self._h, C.c_int(code), out.ctypes.data_as(C.POINTER(C.c_int64))))
        return out

    def localStateIndex(self, nGlobalCells, nGlobalFaces, turbulent=True, compressible=False):
        """Indices into the global state vector (reference ordering) of this rank's local state vector."""
        cg = self.getLocalToGlobal("cells")
        fg = self.getLocalToGlobal("faces")
        ns = 4 + int(bool(turbulent)) + int(bool(compressible))
        parts = [(3 * cg[:, None] + np.arange(3)[None, :]).ravel(), 3 * nGlobalCells + cg]
        if compressible:
            parts.append(4 * nGlobalCells + cg)
        if turbulent:
            parts.append((ns - 1) * nGlobalCells + cg)
        parts.append(ns * nGlobalCells + fg)
        return np.concatenate(parts)

    def setSolverInput(self, inputName, inputType, inputSize, inputs, seeds=None):
        inputs = np.ascontiguousarray(inputs, dtype=np.float64)
        assert len(inputs) == inputSize, "invalid input array size!"
        self._raise(self._L.dab_set_solver_input(self._h, inputName.encode(), inputType.encode(), C.c_int(inputSize), _dp(inputs), None))

    def solvePrimal(self):
        """SIMPLE iterations from the current states (reference pyDASolvers.pyx solvePrimal -> DASimpleFoam::solvePrimal).
        Returns 0 (converged within primalMinResTolDiff of primalMinResTol) or 1; statistics in self.primalStats."""
        fail = C.c_int(1)
        st = PrimalStats()
        self._raise(self._L.dab_solve_primal(self._h, C.byref(fail), C.byref(st)))
        self.primalStats = st
        self._prevPrimalSolTime = getattr(self, "_prevPrimalSolTime", 0.0) + st.iterations * self.getDeltaT()
        return int(fail.value)

    def updateDAOption(self, pyOptions):
        self._options.update(pyOptions)
        self._raise(self._L.dab_update_options(self._h, json.dumps(pyOptions).encode()))

    def updateOFFields(self, states):
        _check_array(states, self.getNLocalAdjointStates(), "states")
        self._raise(self._L.dab_update_of_fields(self._h, _dp(states)))

    def getOFFields(self, states):
        _check_array(states, self.getNLocalAdjointStates(), "states")
        self._raise(self._L.dab_get_of_fields(self._h, _dp(states)))

    def getOFMeshPoints(self, points):
        _check_array(points, self.getNLocalPoints() * 3, "points")
        self._raise(self._L.dab_get_of_mesh_points(self._h, _dp(points)))

    def writeAdjointFields(self, function, writeTime, psi):
        _check_array(psi, self.getNLocalAdjointStates(), "psi")
        self._raise(self._L.dab_write_adjoint_fields(self._h, function.encode(), C.c_double(writeTime), _dp(psi)))

    def writeFields(self, writeTime):
        """The current states as OpenFOAM field files under <case>/<writeTime>/ (runTime.write() of the primal solver)."""
        self._raise(self._L.dab_write_fields(self._h, C.c_double(writeTime)))

    def updateOFMesh(self, points):
        _check_array(points, 3 * self.getNLocalPoints(), "points")
        self._raise(self._L.dab_update_of_mesh(self._h, _dp(points)))

    def getOFField(self, fieldName, fieldType, field):
        n = self.getNLocalCells() * (3 if fieldType == "vector" else 1)
        _check_array(field, n, "field")
        self._raise(self._L.dab_get_of_field(self._h, fieldName.encode(), fieldType.encode(), _dp(field)))

    def getResiduals(self, residuals, isPC=0):
        _check_array(residuals, self.getNLocalAdjointStates(), "residuals")
        self._raise(self._L.dab_get_residuals(self._h, C.c_int(isPC), _dp(residuals)))

    def getInputSize(self, inputName, inputType):
        v = C.c_int64()
        self._raise(self._L.dab_get_input_size(self._h, inputName.encode(), inputType.encode(), C.byref(v)))
        return int(v.value)

    def getOutputSize(self, outputName, outputType):
        v = C.c_int64()
        self._raise(self._L.dab_get_output_size(self._h, outputName.encode(), outputType.encode(), C.byref(v)))
        return int(v.value)

    def getInputDistributed(self, inputName, inputType):
        return 1 if inputType in ("stateVar", "volCoord") else 0

    def getOutputDistributed(self, outputName, outputType):
        return 1 if outputType in ("residual", "forceCouplingOutput") else 0

    def calcJacTVecProduct(self, inputName, inputType, inputs, outputName, outputType, seeds, product):
        inputSize = self.getInputSize(inputName, inputType)
        outputSize = self.getOutputSize(outputName, outputType)
        _check_array(inputs, inputSize, "input")
        _check_array(seeds, outputSize, "seed")
        _check_array(product, inputSize, "product")
        self._raise(self._L.dab_calc_jac_t_vec_product(self._h, inputName.encode(), inputType.encode(), _dp(inputs),
                                                       outputName.encode(), outputType.encode(), _dp(seeds), _dp(product)))

    def calcFunction(self, functionName):
        v = C.c_double()
        self._raise(self._L.dab_calc_function(self._h, functionName.encode(), C.byref(v)))
        return float(v.value)

    def calcOutput(self, outputName, outputType, output):
        """output[:] = the value of one output object (reference pyDASolvers.pyx calcOutput -> DAOutput::run;
        DAOutputFunction.C, DAOutputResidual.C, DAOutputForceCoupling.C).  forceCouplingOutput: the nodal wall forces
        (x, y, z per node) of this rank's faces on the output's patches, in the order of getForceCouplingPoints."""
        _check_array(output, self.getOutputSize(outputName, outputType), "output")
        if outputType == "function":
            output[0] = self.calcFunction(outputName)
        elif outputType == "residual":
            self.getResiduals(output)
        elif outputType == "forceCouplingOutput":
            self._raise(self._L.dab_calc_output(self._h, outputName.encode(), outputType.encode(), _dp(output)))
        else:
            raise DAB200Error("calcOutput: output type %s is not supported (function, residual, forceCouplingOutput)" % outputType)

    def getForceCouplingPoints(self, outputName):
        """The global point index of every node of a forceCouplingOutput, in output order: patches sorted by name, each patch's
        points in ascending order (a point shared by two patches appears once per patch; on several ranks, a point on a partition
        seam appears on every rank with faces around it)."""
        out = np.zeros(self.getOutputSize(outputName, "forceCouplingOutput") // 3, dtype=np.int64)
        self._raise(self._L.dab_get_output_points(self._h, outputName.encode(), out.ctypes.data_as(C.POINTER(C.c_int64))))
        return out

    def calcPrimalResidualStatistics(self, mode):
        """Norm2 / mean / max of every residual block of this rank, and the total norm (reference DASolver.C:745-1000).
        mode "print" also prints them in the reference's format; returns {stateName: {"norm2","mean","max"}, "total": norm2}."""
        if mode not in ("print", "calc"):
            raise DAB200Error("mode not valid")
        n, nC = self.getNLocalAdjointStates(), self.getNLocalCells()
        res = np.zeros(n)
        self.getResiduals(res)
        blocks = {"U": res[:3 * nC].reshape(nC, 3)}
        off, nCellStates = 3 * nC, (n - self.getNLocalFaces()) // nC
        comp = self._solverName != "DASimpleFoam"
        names = (["p", "T"] if comp else ["p"]) + (["nuTilda"] if nCellStates == (6 if comp else 5) else [])
        for nm in names:
            blocks[nm] = res[off:off + nC]
            off += nC
        blocks["phi"] = res[off:]
        out, total = {}, 0.0
        for nm, r in blocks.items():
            a = np.abs(r)
            st = {"norm2": np.sqrt((r * r).sum(axis=0)), "mean": a.mean(axis=0), "max": a.max(axis=0)}
            total += float((r * r).sum())
            out[nm] = st
            if mode == "print":
                for key, label in (("norm2", "Norm2"), ("mean", "Mean"), ("max", "Max")):
                    v = st[key]
                    txt = "(%s)" % " ".join("%g" % x for x in v) if np.ndim(v) else "%g" % v
                    print("%s Residual %s: %s" % (nm, label, txt))
        out["total"] = float(np.sqrt(total))
        if mode == "print":
            print("Total Residual Norm2: %g" % out["total"])
        return out

    def updateStateBoundaryConditions(self):
        """Reference DASolver.C:2863-2886 re-evaluates BCs, nut and the thermo fields after a state change.  Here they are
        functions evaluated inside the kernels from the current states, so there is nothing stored to refresh."""
        return None

    def updateBoundaryConditions(self, fieldName, fieldType):
        """Reference DASolver.C:2814-2845 (correctBoundaryConditions of one field): same remark as above."""
        if fieldType not in ("scalar", "vector"):
            raise DAB200Error("%s not support. Options are: vector or scalar " % fieldType)
        return None

    # ---- mesh quality, mesh / state files, sensitivity maps (pyDASolvers.pyx:320-321, 382-395, 421-462)
    def checkMesh(self):
        """1 if the mesh passes the quality checks of DACheckMesh (thresholds: option checkMeshThreshold, defaults of
        reference pyDAFoam.py:611-616), else 0; the measured values are kept in self.meshQuality."""
        th = dict(maxAspectRatio=1000.0, maxNonOrth=70.0, maxSkewness=4.0, maxIncorrectlyOrientedFaces=0)
        th.update(self._options.get("checkMeshThreshold", {}) or {})
        ok = C.c_int(0)
        rep = (C.c_double * 11)()
        self._raise(self._L.dab_check_mesh(self._h, C.c_double(th["maxNonOrth"]), C.c_double(th["maxSkewness"]), C.c_double(th["maxAspectRatio"]),
                                           C.c_int(int(th["maxIncorrectlyOrientedFaces"])), C.byref(ok), rep))
        keys = ("maxNonOrth", "avgNonOrth", "maxSkewness", "maxAspectRatio", "minVolume", "minFaceArea", "maxOpenness", "nSevereNonOrth",
                "nErrorNonOrth", "nNegativePyramids", "nFailedChecks")
        self.meshQuality = dict(zip(keys, [float(v) for v in rep]))
        return int(ok.value)

    def readStateVars(self, timeVal, timeLevel=0):
        """Fields of <case>/<timeVal>/ -> states.  timeLevel > 0 (old-time levels) belongs to the unsteady solvers."""
        if timeLevel != 0:
            raise DAB200Error("readStateVars: old-time levels belong to the unsteady solvers (not built)")
        self._raise(self._L.dab_read_state_vars(self._h, C.c_double(timeVal)))

    def readMeshPoints(self, timeVal):
        self._raise(self._L.dab_read_mesh_points(self._h, C.c_double(timeVal)))

    def writeMeshPoints(self, points, timeVal):
        _check_array(points, self.getNLocalPoints() * 3, "points")
        name = ("%.6g" % timeVal) if not isinstance(timeVal, str) else timeVal
        self._raise(self._L.dab_write_mesh_points(self._h, _dp(points), name.encode()))

    def writeCurrentMeshPointsToConstant(self):
        self._raise(self._L.dab_write_mesh_points(self._h, None, b"constant"))

    def writeFailedMesh(self, timeVal=9999):
        """The current points under a far time directory for inspection (reference DASolver::writeFailedMesh writes the failed mesh
        to the time the option writeMinorIterations / failed-mesh logic selects; the default here is 9999)."""
        self._raise(self._L.dab_write_mesh_points(self._h, None, ("%.6g" % timeVal).encode()))

    def writeSensMapSurface(self, name, dFdXs, Xs, size, timeName):
        _check_array(dFdXs, size, "dFdXs")
        _check_array(Xs, size, "Xs")
        nrm = C.c_double(0.0)
        self._raise(self._L.dab_write_sens_map_surface(self._h, name.encode(), _dp(dFdXs), _dp(Xs), C.c_int(size), C.c_double(timeName),
                                                       C.byref(nrm)))
        return float(nrm.value)

    def writeSensMapField(self, name, dFdField, fieldType, timeName):
        if fieldType not in ("scalar", "vector"):
            raise DAB200Error("fieldType can be either scalar or vector")
        _check_array(dFdField, self.getNLocalCells() * (3 if fieldType == "vector" else 1), "dFdField")
        self._raise(self._L.dab_write_sens_map_field(self._h, name.encode(), _dp(dFdField), fieldType.encode(), C.c_double(timeName)))

    # ---- index and bookkeeping queries
    def getNLocalAdjointBoundaryStates(self):
        """(3 nVolVectorStates + nVolScalarStates + nModelStates) * nLocalBoundaryFaces (reference DAIndex.C:105-107)."""
        nCellStates = (self.getNLocalAdjointStates() - self.getNLocalFaces()) // self.getNLocalCells()
        return nCellStates * (self.getNLocalFaces() - self.getNLocalInternalFaces())

    def setGlobalXvOffset(self, offset):
        """Offset added to the volCoord indices (default 0).  Every rank holds the full point list and its volCoord products are
        summed over the ranks (the distributed-input convention), so the index of a point is the same on every rank; a caller that
        lays the ranks' point vectors end to end passes the sum of 3*nLocalPoints over the lower ranks instead."""
        self._xvOffset = int(offset)

    def getGlobalXvIndex(self, pointI, coordI):
        """Reference DAIndex.C:704-733: offset + pointI*3 + coordI."""
        assert 0 <= pointI < self.getNLocalPoints() and 0 <= coordI < 3
        return getattr(self, "_xvOffset", 0) + 3 * pointI + coordI

    def getOFFieldGlobal(self, fieldName, fieldType, field):
        """globalField[globalCell] = localField[localCell] for this rank's cells (reference DASolver.C:4484-4517, scalar fields only);
        the entries of other ranks are left untouched, as in the reference (the caller reduces)."""
        if fieldType != "scalar":
            raise DAB200Error("fieldType not valid")
        assert len(field) == self.getNGlobalCells(), "invalid array size!"
        loc = np.zeros(self.getNLocalCells())
        self.getOFField(fieldName, fieldType, loc)
        field[self.getLocalToGlobal("cells")] = loc

    def getInitStateVals(self, printInfo=0):
        """Average of every cell state over the mesh (reference DASolver::getInitStateVals, DASolver.C:3637-3710): U0, U1, U2, p, [T],
        [nuTilda] in self.initStateVals.  On several ranks each rank holds its own share sum(local)/nGlobalCells (the reference reduces
        them with MPI; the caller owns the communicator here)."""
        n, nC, nG = self.getNLocalAdjointStates(), self.getNLocalCells(), self.getNGlobalCells()
        W = np.zeros(n)
        self.getOFFields(W)
        nCellStates = (n - self.getNLocalFaces()) // nC
        comp = self._solverName != "DASimpleFoam"
        names = ["p"] + (["T"] if comp else []) + (["nuTilda"] if nCellStates - 4 - int(comp) > 0 else [])
        vals = {"U%d" % i: float(W[i:3 * nC:3].sum() / nG) for i in range(3)}
        for k, name in enumerate(names):
            vals[name] = float(W[(3 + k) * nC:(4 + k) * nC].sum() / nG)
        self.initStateVals = vals
        if printInfo:
            print("initStateVals: %s" % vals)
        return vals

    def setPrimalBoundaryConditions(self, printInfo=1):
        """Re-apply the primalBC option (reference DASolver::setPrimalBoundaryConditions -> DAField::setPrimalBoundaryConditions)."""
        pbc = self._options.get("primalBC", {})
        if pbc:
            self._raise(self._L.dab_update_options(self._h, json.dumps(dict(primalBC=pbc)).encode()))
        if printInfo and pbc:
            print("Setting primal boundary conditions: %s" % ", ".join(sorted(pbc)))

    def getdFScaling(self, functionName, timeIdx=-1):
        """Weight of a time instance in a time-averaged function (reference DASolver::getdFScaling): steady solvers have one
        instance, weight 1."""
        if functionName not in (self._options.get("function", {}) or {}):
            raise DAB200Error("function %s not found in the function option" % functionName)
        return 1.0

    def meanStatesToStates(self):
        raise DAB200Error("meanStatesToStates (option useMeanStates: step-averaged states of a limit-cycling primal) is not built")

    def hasVolCoordInput(self):
        """1 if any inputInfo entry is of type volCoord (reference DASolver::hasVolCoordInput)."""
        info = self._options.get("inputInfo", {}) or {}
        return int(any(isinstance(v, dict) and v.get("type") == "volCoord" for v in info.values()))

    def getElapsedClockTime(self):
        return time.time() - self._t0Clock

    def getElapsedCpuTime(self):
        return time.process_time() - self._t0Cpu

    # steady solvers: the "time" is the SIMPLE iteration counter of system/controlDict (reference runTime bookkeeping)
    def _controlDict(self):
        if not hasattr(self, "_ctl"):
            self._ctl = {}
            path = os.path.join(self._caseDir, "system", "controlDict")
            if os.path.exists(path):
                for line in open(path):
                    t = line.split("//")[0].strip().rstrip(";").split()
                    if len(t) == 2:
                        self._ctl[t[0]] = t[1]
        return self._ctl

    def getDeltaT(self):
        return float(self._controlDict().get("deltaT", 1.0))

    def getEndTime(self):
        return float(self._controlDict().get("endTime", 0.0))

    def getDdtSchemeOrder(self):
        """Steady solvers run ddtSchemes steadyState; the reference returns 1 for Euler and 2 for backward (unsteady only)."""
        return 1

    def setTime(self, time_, timeIndex):
        self._time, self._timeIndex = float(time_), int(timeIndex)

    def getPrevPrimalSolTime(self):
        return getattr(self, "_prevPrimalSolTime", 0.0)

    def getLatestTime(self):
        """Largest numeric time directory of the case (reference runTime.times().last())."""
        best = 0.0
        for d in os.listdir(self._caseDir):
            try:
                v = float(d)
            except ValueError:
                continue
            if os.path.isdir(os.path.join(self._caseDir, d)):
                best = max(best, v)
        return best

    def runFPAdj(self, dFdW, psi):
        """Fixed-point adjoint (reference pyDASolvers.pyx:412-413, DASimpleFoam::runFPAdj): stationary iteration from psi = 0 with
        adjEqnOption fpMaxIters / fpRelTol / fpMinResTolDiff and the reference's termination rule; the approximate inverse is this
        engine's preconditioner (include/dab200.h dab_run_fp_adj).  Returns 0 (converged, possibly by the relaxed rule) or 1."""
        n = self.getNLocalAdjointStates()
        _check_array(dFdW, n, "dFdW")
        _check_array(psi, n, "psi")
        fail = C.c_int(1)
        st = KspStats()
        self._raise(self._L.dab_run_fp_adj(self._h, _dp(dFdW), _dp(psi), C.byref(fail), C.byref(st)))
        self.fpStats = st
        return int(fail.value)

    def solveAdjointFP(self, dFdW, psi):
        return self.runFPAdj(dFdW, psi)

    def printAllOptions(self):
        """Reference DASolver.H printAllOptions: dump the options dictionary."""
        print(json.dumps(self._options, indent=2, sort_keys=True, default=str))

    def runColoring(self):
        # the colouring is computed inside calcdRdWT on first use (reference DASolver.C:708-743)
        return None

    def calcdRdWT(self, isPC, dRdWT):
        assert isPC == 1, "only the preconditioner matrix (isPC=1) is assembled explicitly; dRdWT itself is matrix-free"
        self._raise(self._L.dab_calc_drdwt_pc(self._h))
        dRdWT.assembled = True
        wj = self._options.get("writeJacobians", [])
        if "dRdWTPC" in wj or "all" in wj:
            # DAUtility::writeMatrixBinary(dRdWT, "dRdWTPC") (reference DASolver.C:1080-1085): PETSc binary AIJ in the case directory
            from . import petsc_io
            rp, cl, vl = self.getPCMatrix()
            name = "dRdWTPC.bin" if self._nRanks == 1 else "dRdWTPC_rank%d.bin" % self._rank
            petsc_io.write_mat(os.path.join(self._caseDir, name), rp, cl, vl)

    def calcPCMatWithFvMatrix(self, PCMat, turbOnly=0):
        """Reference pyDASolvers.pyx calcPCMatWithFvMatrix -> DASolver::calcPCMatWithFvMatrix (DASolver.C:2888-2988): the turbulence
        block of the preconditioner from the relaxed nuTilda fvMatrix; entries land in PCMat (INSERT_VALUES semantics)."""
        nnz = C.c_int64()
        self._raise(self._L.dab_calc_pc_mat_fvmatrix(self._h, C.c_int(int(turbOnly)), C.byref(nnz), None, None, None))
        rows, cols, vals = np.zeros(nnz.value, dtype=np.int32), np.zeros(nnz.value, dtype=np.int32), np.zeros(nnz.value)
        if nnz.value:
            self._raise(self._L.dab_calc_pc_mat_fvmatrix(self._h, C.c_int(int(turbOnly)), C.byref(nnz), rows.ctypes.data_as(C.POINTER(C.c_int32)),
                                                         cols.ctypes.data_as(C.POINTER(C.c_int32)), _dp(vals)))
        if PCMat.vals is None:
            PCMat.rows, PCMat.cols, PCMat.vals = rows, cols, vals
        else:  # INSERT_VALUES over what is there: new entries replace old ones at the same position
            key_old = PCMat.rows.astype(np.int64) << 32 | PCMat.cols.astype(np.int64)
            key_new = rows.astype(np.int64) << 32 | cols.astype(np.int64)
            keep = ~np.isin(key_old, key_new)
            PCMat.rows = np.concatenate([PCMat.rows[keep], rows])
            PCMat.cols = np.concatenate([PCMat.cols[keep], cols])
            PCMat.vals = np.concatenate([PCMat.vals[keep], vals])
        PCMat.assembled = True

    def getPCMatrixSize(self):
        """(rows, stored entries) of the dRdWTPC pattern of the last calcdRdWT(1, ...)."""
        n, nnz = C.c_int64(), C.c_int64()
        self._raise(self._L.dab_get_pc_matrix(self._h, C.byref(n), C.byref(nnz), None, None, None))
        return int(n.value), int(nnz.value)

    def getPCMatrix(self):
        """(row_ptr, cols, vals) of the assembled dRdWTPC (CSR, external numbering); needs "dRdWTPC" in writeJacobians."""
        n, nnz = C.c_int64(), C.c_int64()
        self._raise(self._L.dab_get_pc_matrix(self._h, C.byref(n), C.byref(nnz), None, None, None))
        rp, cl, vl = np.zeros(n.value + 1, dtype=np.int64), np.zeros(nnz.value, dtype=np.int32), np.zeros(nnz.value)
        self._raise(self._L.dab_get_pc_matrix(self._h, C.byref(n), C.byref(nnz), rp.ctypes.data_as(C.POINTER(C.c_int64)),
                                              cl.ctypes.data_as(C.POINTER(C.c_int32)), _dp(vl)))
        return rp, cl[:nnz.value], vl[:nnz.value]

    def getPCFactors(self):
        """Test hook: (row_ptr, cols, vals, perm, colour) of the ILU(0) factors of the last calcdRdWT(1, ...) in factorisation order
        (CSR, sorted columns): L multipliers left of the diagonal, the stored 1/u_ii on it, U right of it, as the triangular solves
        read them; perm[new] = external state index, colour[new] = ordering colour of the row."""
        n, nnz = C.c_int64(), C.c_int64()
        self._raise(self._L.dab_get_pc_factors(self._h, C.byref(n), C.byref(nnz), None, None, None, None, None))
        rp, cl, vl = np.zeros(n.value + 1, dtype=np.int64), np.zeros(nnz.value, dtype=np.int32), np.zeros(nnz.value)
        perm, colour = np.zeros(n.value, dtype=np.int32), np.zeros(n.value, dtype=np.int32)
        ip = C.POINTER(C.c_int32)
        self._raise(self._L.dab_get_pc_factors(self._h, C.byref(n), C.byref(nnz), rp.ctypes.data_as(C.POINTER(C.c_int64)),
                                               cl.ctypes.data_as(ip), _dp(vl), perm.ctypes.data_as(ip), colour.ctypes.data_as(ip)))
        return rp, cl[:nnz.value], vl[:nnz.value], perm, colour

    def getPCAggregates(self):
        """Test hook: the global aggregate id of every local cell of the preconditioner's pressure coarse space."""
        agg = np.zeros(self.getNLocalCells(), dtype=np.int32)
        self._raise(self._L.dab_get_pc_aggregates(self._h, agg.ctypes.data_as(C.POINTER(C.c_int32))))
        return agg

    def getFaceLoopWidth(self):
        """Test hook: 6 when the cell-per-thread kernels run the unrolled six-face loops, 0 for the rolled loops."""
        nf = C.c_int()
        self._raise(self._L.dab_get_face_loop_width(self._h, C.byref(nf)))
        return nf.value

    def getTransonicPressureSystem(self, coarse=True, rc=None):
        """Test hook: the transonic pressure equation of the current state (DATurboFoam, SIMPLE { transonic yes; }) as the first SIMPLE
        iteration assembles it, and one BiCGStab solve of it from the current p; the states are not changed.  Returns a dict with the
        ELL rows (nbr, off: [maxCF, nC]; diag, b: [nC]), the solution x, the iteration count, agg_of (local aggregate per cell, -1
        without coarse space) and, when rc is given and the coarse space is on, yc = Ac^-1 rc from the solver's coarse apply."""
        mcf, nagg = C.c_int(), C.c_int()
        nil = None
        self._raise(self._L.dab_transonic_pressure_probe(self._h, C.c_int(int(coarse)), C.byref(mcf), C.byref(nagg), nil, nil, nil, nil, nil,
                                                         nil, nil, nil, nil))
        nC = self.getNLocalCells()
        ip = C.POINTER(C.c_int32)
        nbr, off = np.zeros(mcf.value * nC, dtype=np.int32), np.zeros(mcf.value * nC)
        diag, b, x, agg = np.zeros(nC), np.zeros(nC), np.zeros(nC), np.zeros(nC, dtype=np.int32)
        its = C.c_int()
        yc, rcp = None, None
        if rc is not None:  # the first n_agg entries are used
            assert len(rc) >= nagg.value, "rc needs n_agg = %d entries" % nagg.value
            rc = np.ascontiguousarray(rc[:nagg.value], dtype=np.float64)
            yc, rcp = np.zeros(nagg.value), _dp(rc)
        self._raise(self._L.dab_transonic_pressure_probe(self._h, C.c_int(int(coarse)), C.byref(mcf), C.byref(nagg), nbr.ctypes.data_as(ip),
                                                         _dp(off), _dp(diag), _dp(b), _dp(x), C.byref(its), agg.ctypes.data_as(ip), rcp,
                                                         _dp(yc) if yc is not None else None))
        return dict(nbr=nbr.reshape(mcf.value, nC), off=off.reshape(mcf.value, nC), diag=diag, b=b, x=x, iterations=its.value, agg_of=agg,
                    n_agg=nagg.value, yc=yc)

    def initializedRdWTMatrixFree(self):
        return None

    def destroydRdWTMatrixFree(self):
        return None

    def createMLRKSPMatrixFree(self, jacPCMat, myKSP):
        assert jacPCMat.assembled, "call calcdRdWT(1, dRdWTPC) first"
        myKSP.ready = True

    def updateKSPPCMat(self, PCMat, myKSP):
        myKSP.ready = PCMat.assembled

    def solveLinearEqn(self, myKSP, rhsVec, solVec):
        n = self.getNLocalAdjointStates()
        _check_array(rhsVec, n, "rhs")
        _check_array(solVec, n, "sol")
        fail = C.c_int(1)
        st = KspStats()
        self._raise(self._L.dab_solve_linear_eqn(self._h, _dp(rhsVec), _dp(solVec), C.byref(fail), C.byref(st)))
        if myKSP is not None:
            myKSP.stats = st
        return int(fail.value)

    def applyPC(self, v, z):
        n = self.getNLocalAdjointStates()
        _check_array(v, n, "v")
        _check_array(z, n, "z")
        self._raise(self._L.dab_pc_apply(self._h, _dp(v), _dp(z)))

    # ---- v2/v3-era names used by BASELINE.json's north_star (thin aliases)
    def calcdRdWTPsiAD(self, psi, dRdWTPsi):
        n = self.getNLocalAdjointStates()
        _check_array(psi, n, "psi")
        _check_array(dRdWTPsi, n, "dRdWTPsi")
        self._raise(self._L.dab_drdwt_mat_vec(self._h, _dp(psi), _dp(dRdWTPsi)))

    def solveAdjoint(self, dFdW, psi):
        ksp = KSP()
        return self.solveLinearEqn(ksp, dFdW, psi), ksp.stats

    # ---- measurement hooks
    def benchDevice(self, which, n):
        ms = C.c_double()
        nl = C.c_int64()
        self._raise(self._L.dab_bench_device(self._h, C.c_int(which), C.c_int(n), C.byref(ms), C.byref(nl)))
        return float(ms.value), int(nl.value)

    def benchSetVector(self, x):
        _check_array(x, self.getNLocalAdjointStates(), "x")
        self._raise(self._L.dab_bench_set_vector(self._h, _dp(x)))

    def algorithmicBytes(self, which=0):
        v = C.c_int64()
        self._raise(self._L.dab_algorithmic_bytes(self._h, C.c_int(which), C.byref(v)))
        return int(v.value)
