"""PYDAFOAM -- the user-facing class of the reference (dafoam/pyDAFoam.py:673-2200) for the path this package covers,
on top of the GPU engine: primal (`__call__`), functions, states / volume coordinates, residuals, and the discrete
adjoint with its total derivatives (what `DAFoamSolver.solve_linear` / `apply_linear` and `DAFoamFunctions.
compute_jacvec_product` do in dafoam/mphys/mphys_dafoam.py:405-574, 778-792 -- and what the v2/v3 API exposed as
`solveAdjoint` / `calcTotalDeriv`).

Not reproduced (out of scope, SURVEY.md section 8): OpenMDAO/MPhys components, pyGeo/IDWarp hooks, family groups and
surface maps, decomposePar, option type checking.  There is no CPU fallback: constructing the object needs
libdab200.so and a CUDA GPU (sm_90a)."""
from __future__ import annotations

import copy

import numpy as np

from .pyDASolvers import KSP, Mat, pyDASolvers

# the subset of DAOPTION (reference dafoam/pyDAFoam.py:39-662) this engine reads, with the reference's defaults
DEFAULT_OPTIONS = {
    "solverName": "DASimpleFoam",
    "primalMinResTol": 1.0e-8,
    "primalMinResTolDiff": 1.0e2,
    "primalMinIters": 1,
    "function": {},
    "inputInfo": {},
    "normalizeStates": {},
    "normalizeResiduals": ["URes", "pRes", "nuTildaRes", "phiRes"],
    "useConstrainHbyA": True,
    "adjPartDerivFDStep": {"State": 1.0e-6},
    "adjEqnOption": {"gmresRelTol": 1.0e-6, "gmresAbsTol": 1.0e-14, "gmresMaxIters": 1000, "gmresRestart": 1000,
                     "gmresTolDiff": 1.0e2, "useMGSO": False, "printInfo": 0},
    "adjPCLag": 10000,
    "printInterval": 100,
}


class Error(Exception):
    """Fatal error of the wrapper (reference dafoam/pyDAFoam.py:2296-2316)."""


class AnalysisError(Exception):
    """OpenMDAO's AnalysisError role (reference mphys_dafoam.py:329, 346, 557): a recoverable failure the optimiser may step back from."""


class PYDAFOAM:
    def __init__(self, comm=None, options=None, caseDir=".", device=0, _lib_path=None):
        """options: the daOptions dict of a run script; caseDir replaces the reference's implicit os.getcwd().
        `comm` is accepted for signature compatibility (one process per GPU; see pyDASolvers for the multi-rank form)."""
        if options is None:
            raise Error("The 'options' keyword argument must be passed pyDAFoam.")
        self.comm = comm
        self.dtype = "d"
        self.options = copy.deepcopy(DEFAULT_OPTIONS)
        for k, v in options.items():
            if isinstance(v, dict) and isinstance(self.options.get(k), dict):
                self.options[k] = dict(self.options[k], **v)
            else:
                self.options[k] = v
        args = "%s -python" % self.options["solverName"]
        self.solver = pyDASolvers(args, self.options, caseDir=caseDir, device=device, _lib_path=_lib_path)  # _lib_path: test-suite only
        self.solverAD = self.solver  # one engine: the reverse sweep is hand-derived, there is no separate AD build
        self.nSolvePrimals = 1
        self.nSolveAdjoints = 1
        self.primalFail = 0
        self.adjointFail = 0
        self._pc = None
        self._ksp = None
        self._psi = {}
        # adjPCLag bookkeeping of DAFoamSolver.solve_linear (reference mphys_dafoam.py:481-514): `solution_counter` advances once per
        # design iteration IN WHICH DERIVATIVES ARE ASKED FOR (the first adjoint after a new primal solution, `renamed`), not per primal
        # solution -- line-search primals do not age the preconditioner; it is re-assembled when (solution_counter - 1) % adjPCLag == 0
        self.solution_counter = 1
        self._renamed = True  # a primal solution not yet followed by an adjoint
        self.nPCAssemblies = 0

    # ---- options -----------------------------------------------------------------------------------------
    def getOption(self, name):
        if name not in self.options:
            raise Error("%s is not a valid option name." % name)
        return self.options[name]

    def setOption(self, name, value):
        if isinstance(value, dict) and isinstance(self.options.get(name), dict):
            self.options[name] = dict(self.options[name], **value)
        else:
            self.options[name] = value

    def updateDAOption(self):
        self.solver.updateDAOption(self.options)

    # ---- primal --------------------------------------------------------------------------------------------
    def __call__(self):
        """Solve the primal (reference pyDAFoam.py:800-821)."""
        self.primalFail = self.solver.solvePrimal()
        self.nSolvePrimals += 1
        self._renamed = True  # the next adjoint opens a new derivative iteration (adjPCLag counts those)
        self._psi = {}

    def solve_nonlinear(self, inputs=None):
        """The body of DAFoamSolver.solve_nonlinear (reference mphys_dafoam.py:314-368) without the OpenMDAO vectors: assign the
        solver inputs, refuse a mesh that fails checkMesh (the failed mesh is written for inspection), honour prepareCaseOnly,
        solve the primal, raise AnalysisError when it fails, print the residual statistics, and return the states."""
        if inputs:
            self.set_solver_input(inputs)
        if self.solver.checkMesh() != 1:
            self.solver.writeFailedMesh()
            raise AnalysisError("Mesh quality error!")
        if self.options.get("prepareCaseOnly", False):
            self.solver.writeCurrentMeshPointsToConstant()
            return None
        self()
        if self.primalFail != 0:
            raise AnalysisError("Primal solution failed!")
        self.solver.calcPrimalResidualStatistics("print")
        return self.getStates()

    def evalFunctions(self, funcs):
        """funcs[name] = value for every entry of the `function` option (reference pyDAFoam.py:917-939)."""
        for funcName in list(self.getOption("function").keys()):
            funcs[funcName] = self.solver.calcFunction(funcName)

    def set_solver_input(self, inputs, DVGeo=None):
        """Assign the inputs attached to the solver component (reference pyDAFoam.py:1350-1374)."""
        inputDict = self.getOption("inputInfo")
        for inputName in list(inputDict.keys()):
            if "solver" in inputDict[inputName].get("components", ["solver"]) and inputName in inputs:
                x = np.ascontiguousarray(inputs[inputName], dtype=np.float64)
                self.solver.setSolverInput(inputName, inputDict[inputName]["type"], len(x), x, np.zeros(len(x)))

    # ---- sizes, states, coordinates, residuals (reference pyDAFoam.py:2078-2130) ---------------------------
    def getNLocalAdjointStates(self):
        return self.solver.getNLocalAdjointStates()

    def getNLocalPoints(self):
        return self.solver.getNLocalPoints()

    def getStates(self):
        states = np.zeros(self.solver.getNLocalAdjointStates(), self.dtype)
        self.solver.getOFFields(states)
        return states

    def setStates(self, states):
        self.solver.updateOFFields(np.ascontiguousarray(states, dtype=np.float64))
        self._pc = None
        self._psi = {}
        self._renamed = True

    def getVolCoords(self):
        xv = np.zeros(3 * self.solver.getNLocalPoints(), self.dtype)
        self.solver.getOFMeshPoints(xv)
        return xv

    def setVolCoords(self, vol_coords):
        self.solver.updateOFMesh(np.ascontiguousarray(vol_coords, dtype=np.float64))
        self._psi = {}  # the preconditioner is kept: it is refreshed every adjPCLag primal solutions

    def getResiduals(self):
        residuals = np.zeros(self.solver.getNLocalAdjointStates(), self.dtype)
        self.solver.getResiduals(residuals)
        return residuals

    # ---- output --------------------------------------------------------------------------------------------
    def writeFields(self, writeTime=None):
        """The current states as OpenFOAM fields under <case>/<writeTime>/ (what the reference's primal leaves on disk)."""
        self.solver.writeFields(self.nSolvePrimals if writeTime is None else writeTime)

    def writeAdjointFields(self, function, writeTime, psi):
        """adjoint_<function>_<state> fields for post-processing (reference pyDAFoam.py:907-915)."""
        self.solver.writeAdjointFields(function, writeTime, np.ascontiguousarray(psi, dtype=np.float64))

    # ---- adjoint -------------------------------------------------------------------------------------------
    def solveAdjoint(self, functionName):
        """psi of one function: dFdW, preconditioner (re)assembly, GMRES (reference mphys_dafoam.py:433-574).
        Returns psi; self.adjointFail holds the reference's 0/1."""
        n = self.solver.getNLocalAdjointStates()
        W = self.getStates()
        dFdW = np.zeros(n)
        self.solver.calcJacTVecProduct("states", "stateVar", W, functionName, "function", np.array([1.0]), dFdW)
        method = self.options.get("adjEqnSolMethod", "Krylov")
        if method not in ("Krylov", "fixedPoint"):  # reference mphys_dafoam.py:562
            raise RuntimeError("adjEqnSolMethod=%s not valid! Options are: Krylov or fixedPoint" % method)
        renamed = self._renamed
        if renamed:
            self.solution_counter += 1
            self._renamed = False
        adjPCLag = max(1, int(self.getOption("adjPCLag")))
        if self._pc is None or (renamed and (self.solution_counter - 1) % adjPCLag == 0):
            self.nPCAssemblies += 1
            self._pc, self._ksp = Mat(), KSP()
            self.solver.calcdRdWT(1, self._pc)
            self.solver.createMLRKSPMatrixFree(self._pc, self._ksp)
        psi = np.zeros(n)
        if method == "fixedPoint":  # reference mphys_dafoam.py:549-557
            self.adjointFail = self.solver.solveAdjointFP(dFdW, psi)
        else:
            self.adjointFail = self.solver.solveLinearEqn(self._ksp, dFdW, psi)
        self.nSolveAdjoints += 1
        self._psi[functionName] = psi
        return psi

    def calcTotalDeriv(self, functionName, inputName, inputValue=None):
        """dF/dx = dF/dx|_W - [dR/dx]^T psi for one input of `inputInfo` (volCoord, patchVelocity, ...), with the adjoint
        solved on demand (reference mphys_dafoam.py:405-431 apply_linear + :778-792 compute_jacvec_product)."""
        info = self.getOption("inputInfo")[inputName]
        inputType = info["type"]
        if functionName not in self._psi:
            self.solveAdjoint(functionName)
        if self.adjointFail:
            raise Error("the adjoint of %s did not converge" % functionName)
        psi = self._psi[functionName]
        if inputValue is None:
            if inputType == "volCoord":
                inputValue = self.getVolCoords()
            else:
                raise Error("calcTotalDeriv: pass the current value of input %s" % inputName)
        x = np.ascontiguousarray(inputValue, dtype=np.float64)
        dFdx, dRdxTpsi = np.zeros(len(x)), np.zeros(len(x))
        self.solver.calcJacTVecProduct(inputName, inputType, x, functionName, "function", np.array([1.0]), dFdx)
        self.solver.calcJacTVecProduct(inputName, inputType, x, "R", "residual", psi, dRdxTpsi)
        return dFdx - dRdxTpsi
