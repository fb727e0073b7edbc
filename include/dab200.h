/*
 * dab200.h -- C ABI of the GPU-native discrete-adjoint engine (libdab200.so).
 *
 * This is the drop-in boundary for the adjoint hot path of mdolab/dafoam: each entry point replaces
 * one method of the reference's Cython class `pyDASolvers` (reference src/pyDASolvers/pyDASolvers.pyx:
 * 45-114 extern block, class body :117-483) / C++ forwarding class `Foam::DASolvers`
 * (reference src/pyDASolvers/DASolvers.H).  Plain pointers and sizes only; all arrays are
 * caller-allocated HOST buffers of doubles, borrowed for the duration of the call (the same ownership
 * convention as the reference's numpy arguments); the library owns all device memory.
 *
 * Every function returns 0 on success and a non-zero code on error; dab_last_error() returns the
 * message of the last failing call of the calling thread.  The library requires a CUDA device; it
 * never falls back to a CPU path.
 *
 * State-vector layout ("state" ordering, reference src/adjoint/DAIndex/DAIndex.C:188-257):
 *     W = [ U(cell-major xyz) | p | nuTilda (SA only) | phi (internal faces, then boundary faces) ]
 * Residual vectors use the same layout (reference src/adjoint/DAOutput/DAOutputResidual.C:50-118).
 */
#ifndef DAB200_H
#define DAB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dab_solver dab_solver;

/* boundary-condition kinds parsed from the case's 0/<field> files */
enum dab_bc_kind
{
    DAB_BC_FIXED_VALUE = 0,
    DAB_BC_ZERO_GRADIENT = 1,
    DAB_BC_INLET_OUTLET = 2,
    DAB_BC_OUTLET_INLET = 3,
    DAB_BC_SYMMETRY = 4,
    DAB_BC_CALCULATED = 5,
    DAB_BC_NUT_LOW_RE = 6
};

/* statistics of one Krylov solve (reference prints these: src/adjoint/DALinearEqn/DALinearEqn.C:361-418) */
typedef struct dab_ksp_stats
{
    int32_t iterations;
    int32_t converged_reason; /* 2: rtol, 3: atol, -3: max iterations */
    double initial_residual;
    double final_residual;
    double solve_seconds;      /* device time of the GMRES loop */
    double pc_setup_seconds;   /* preconditioner assembly + factorisation */
    int32_t n_matvec;          /* number of dRdWT*psi products */
    int32_t pc_assemblies;     /* preconditioner assemblies of this handle so far (adjPCLag bookkeeping) */
} dab_ksp_stats;

/* per-equation initial residuals of the last SIMPLE iteration (what the reference prints through
 * DAUtility::primalResidualControl, src/adjoint/DAUtility/DAUtility.C:734-801) */
typedef struct dab_primal_stats
{
    int32_t iterations;
    int32_t converged;        /* 1: max residual < primalMinResTol */
    int32_t p_iterations;     /* pressure-solver iterations summed over the run */
    int32_t reserved;
    double max_residual;      /* max over equations (median component for U) */
    double res_u[3];
    double res_p;
    double res_nutilda;
    double seconds;
} dab_primal_stats;

const char* dab_last_error(void);
const char* dab_version(void);

/* DASolvers::DASolvers(char* argsAll, PyObject* pyOptions) + initSolver()
 * (reference pyDASolvers.pyx:136-155, DASolvers.C:15-23, DASolver.C:35-118, DASimpleFoam.C:81-121).
 * case_dir: OpenFOAM case (constant/polyMesh, 0/, constant/, system/); args_all: e.g.
 * "DASimpleFoam -python"; options_json: the DAOPTION dict serialised as JSON
 * (reference dafoam/pyDAFoam.py:39-662 for the keys).  rank/n_ranks/nccl_unique_id describe the
 * domain decomposition (nccl_unique_id may be NULL when n_ranks == 1). device: CUDA ordinal. */
int dab_create(const char* case_dir, const char* args_all, const char* options_json, int device, int rank,
               int n_ranks, const void* nccl_unique_id, dab_solver** out);
int dab_destroy(dab_solver* s);

/* 128-byte NCCL unique id for multi-rank creation (rank 0 calls it, the host broadcasts it) */
int dab_nccl_unique_id(void* out128);

/* local -> global maps of a partitioned case: what = 0 cells [nLocalCells], 1 faces [nLocalFaces],
 * 2 face ownership flags [nLocalFaces] (0: the phi DOF of this cut face lives on the neighbouring rank and the
 * local slot is a structural zero).  Replaces reading processorN/polyMesh/{cell,face}ProcAddressing. */
int dab_get_local_to_global(dab_solver* s, int what, int64_t* out);

/* TEST BUILD ONLY: halo-exchange / all-reduce callbacks used by the next dab_create instead of NCCL
 * (the product build returns an error).  exchange(ctx, nPeers, peers, sendBufs, sendCounts, recvBufs, recvCounts);
 * allreduce(ctx, buf, n) sums n doubles over the ranks in place. */
typedef void (*dab_exchange_cb)(void* ctx, int n_peers, const int* peers, const double* const* send_bufs, const int* send_counts,
                                double* const* recv_bufs, const int* recv_counts);
typedef void (*dab_allreduce_cb)(void* ctx, double* buf, int n);
int dab_set_comm_callbacks(dab_exchange_cb exchange, dab_allreduce_cb allreduce, void* ctx);

/* getNLocalAdjointStates / getNLocalCells / getNGlobalCells / getNLocalPoints (pyDASolvers.pyx) */
int dab_n_local_adjoint_states(dab_solver* s, int64_t* out);
int dab_n_local_cells(dab_solver* s, int64_t* out);
int dab_n_global_cells(dab_solver* s, int64_t* out);
int dab_n_local_points(dab_solver* s, int64_t* out);
/* residual evaluations of one volCoord product (0 before the first product); the same on every rank */
int dab_volcoord_evaluations(dab_solver* s, int64_t* out);
int dab_n_local_faces(dab_solver* s, int64_t* out);
int dab_n_local_internal_faces(dab_solver* s, int64_t* out);

/* updateDAOption(pyOptions) (pyDASolvers.pyx; reference DASolver.H updateDAOption) */
int dab_update_options(dab_solver* s, const char* options_json);

/* updateOFFields(states) / getOFFields(states): DASolver::updateOFFields = state2OFField +
 * updateStateBoundaryConditions (reference DASolver.C:1291-1300, 2863-2886).  Setting the states also
 * records the forward intermediates the matrix-free product reuses (the role of the reference's
 * initializeGlobalADTape4dRdWT, DASolver.C:1411-1441). */
int dab_update_of_fields(dab_solver* s, const double* states);
int dab_get_of_fields(dab_solver* s, double* states);

/* getOFMeshPoints(points) (pyDASolvers.pyx:267-270) */
int dab_get_of_mesh_points(dab_solver* s, double* points);
/* writeAdjointFields(function, writeTime, psi): the adjoint vector as OpenFOAM fields adjoint_<function>_<state> under
 * <case>/<writeTime>/ (reference pyDASolvers.pyx writeAdjointFields, DASolver.C:4055-4160), and the current states the way
 * runTime.write() leaves them (U, p, [T], [nuTilda], phi) -- readable back as a case's 0/ fields. ASCII, one GPU. */
int dab_write_adjoint_fields(dab_solver* s, const char* function, double write_time, const double* psi);
int dab_write_fields(dab_solver* s, double write_time);

/* readStateVars(timeVal, timeLevel) (pyDASolvers.pyx:382-383, DASolver::readStateVars): the fields U, p, [T], [nuTilda] and, when present,
 * phi of <case>/<timeVal>/ become the states (boundary conditions stay those of 0/).  readMeshPoints(timeVal) (pyDASolvers.pyx:385-386):
 * <case>/<timeVal>/polyMesh/points become the mesh points.  writeMeshPoints(points, timeVal) (pyDASolvers.pyx:388-392), also the body of
 * writeCurrentMeshPointsToConstant ("constant") and writeFailedMesh: points == NULL writes the current points. */
int dab_read_state_vars(dab_solver* s, double time_val);
int dab_read_mesh_points(dab_solver* s, double time_val);
int dab_write_mesh_points(dab_solver* s, const double* points, const char* dir_name);
/* writeSensMapSurface(name, dFdXs, Xs, size, timeName) / writeSensMapField(name, dFdField, fieldType, timeName)
 * (pyDASolvers.pyx:421-462, DASolver.C:3840-4053): derivative maps as dimensionless OpenFOAM fields under <case>/<timeName>/ */
int dab_write_sens_map_surface(dab_solver* s, const char* name, const double* dfdxs, const double* xs, int size, double time_name,
                               double* min_distance_norm);
int dab_write_sens_map_field(dab_solver* s, const char* name, const double* dfdfield, const char* field_type, double time_name);
/* checkMesh() (pyDASolvers.pyx:320-321, DACheckMesh.C:45-79, DACheckGeometry.C:256-478): mesh_ok = 1 when no check fails with the
 * thresholds of the option checkMeshThreshold.  report (may be NULL): maxNonOrth, avgNonOrth [deg], maxSkewness, maxAspectRatio,
 * minVolume, minFaceArea, maxOpenness, nSevereNonOrth, nErrorNonOrth, nNegativePyramids, nFailedChecks */
#define DAB_CHECK_MESH_REPORT 11
int dab_check_mesh(dab_solver* s, double max_non_orth, double max_skewness, double max_aspect_ratio, int max_incorrectly_oriented_faces,
                   int* mesh_ok, double* report);

/* updateOFMesh(points): new point coordinates (3*nLocalPoints), geometry recomputed, wall distance frozen
 * (reference pyDASolvers.pyx updateOFMesh, DASolver::updateOFMesh) */
int dab_update_of_mesh(dab_solver* s, const double* points);
/* getOFField(name, type, field): read-only access to a cell field ("U","p","nuTilda","nut","yWall","V") */
int dab_get_of_field(dab_solver* s, const char* name, const char* type, double* field);

/* getResiduals(residuals): R(W) at the current states (reference DASolver.C:2847-2861,
 * DAResidualSimpleFoam.C:106-237, DASpalartAllmaras.C:407-488); is_pc selects the div(pc) schemes. */
int dab_get_residuals(dab_solver* s, int is_pc, double* residuals);

/* calcJacTVecProduct(inputName, inputType, input, outputName, outputType, seed, product)
 * (reference DASolver.C:1690-1839).  Supported pairs: (stateVar -> residual), (stateVar -> function),
 * (stateVar -> forceCouplingOutput), (volCoord -> forceCouplingOutput), and patchVelocity / patchVar /
 * fvSourcePar / volCoord -> residual and function.  A forceCouplingOutput seed has dab_get_output_size
 * entries (this rank's nodes). */
int dab_calc_jac_t_vec_product(dab_solver* s, const char* input_name, const char* input_type, const double* input,
                               const char* output_name, const char* output_type, const double* seed,
                               double* product);

/* Matrix-free product y = diag(n) * (dR/dW)^T x at the current states: the body of the reference's
 * PETSc shell-matrix callback DASolver::dRdWTMatVecMultFunction (DASolver.C:1364-1409);
 * v2/v3-era name: calcdRdWTPsiAD. */
int dab_drdwt_mat_vec(dab_solver* s, const double* x, double* y);

/* calcdRdWT(isPC=1, dRdWTPC) + createMLRKSPMatrixFree(dRdWTPC, ksp): assemble the preconditioner
 * matrix from the first-order residual by coloured finite differences and factorise it
 * (reference DASolver.C:948-1089, DAPartDeriv.C:350-474, DALinearEqn.C:28-339). */
int dab_calc_drdwt_pc(dab_solver* s);

/* z = M^-1 v with the factorised dRdWTPC (the PCApply of the reference's KSP, DALinearEqn.C:142-310) */
int dab_pc_apply(dab_solver* s, const double* v, double* z);

/* solveLinearEqn(ksp, rhs, sol): right-preconditioned restarted GMRES on the device
 * (reference DASolver.C:1121-1155, DALinearEqn.C:341-437).  *fail = 0/1 with the reference's
 * success rule (relRatio > gmresTolDiff && absRatio > gmresTolDiff  =>  1). */
int dab_solve_linear_eqn(dab_solver* s, const double* rhs, double* sol, int* fail, dab_ksp_stats* stats);

/* runFPAdj(dFdW, psi) / solveAdjointFP (pyDASolvers.pyx:412-416; reference DASimpleFoam::runFPAdj, DASimpleFoam.C:189-909): stationary
 * adjoint iteration from psi = 0 with adjEqnOption.fpMaxIters / fpRelTol / fpMinResTolDiff and the reference's per-block termination
 * rule; the approximate inverse is this engine's preconditioner, not the reference's transposed SIMPLE operators.  *fail = 0/1. */
int dab_run_fp_adj(dab_solver* s, const double* dfdw, double* psi, int* fail, dab_ksp_stats* stats);

/* The assembled preconditioner matrix dRdWTPC of this rank as CSR (rows: states, columns: residuals, external numbering,
 * sorted columns) -- the matrix the reference writes with DAUtility::writeMatrixBinary(dRdWT, "dRdWTPC") when the
 * writeJacobians option lists it (DASolver.C:1080-1085, DAUtility.C:411-441).  Call with row_ptr == NULL to get the sizes,
 * then with buffers of n_rows+1 / nnz / nnz entries.  The option writeJacobians must list "dRdWTPC" (or "all") before
 * dab_calc_drdwt_pc, otherwise only the factorisation is kept. */
int dab_get_pc_matrix(dab_solver* s, int64_t* n_rows, int64_t* nnz, int64_t* row_ptr, int32_t* cols, double* vals);

/* Test hook (no counterpart in the reference): the ILU(0) factors of the last dab_calc_drdwt_pc in factorisation order, CSR with
 * sorted columns -- strictly lower entries are the L multipliers, the diagonal holds the stored reciprocal 1/u_ii, upper entries are
 * U; the values the triangular solves read (the fp32 copy widened when adjEqnOption.pcStorage is "fp32").  perm[new] = external
 * state index, colour[new] = ordering colour (level) of the row.  Same two-call size protocol as dab_get_pc_matrix; perm and colour
 * take n_rows entries.  Does not need writeJacobians. */
int dab_get_pc_factors(dab_solver* s, int64_t* n_rows, int64_t* nnz, int64_t* row_ptr, int32_t* cols, double* vals, int32_t* perm,
                       int32_t* colour);

/* Test hook (no counterpart in the reference): the global aggregate id of every local cell of the preconditioner's pressure coarse
 * space (adjEqnOption.coarseAggregates > 0); an error without a coarse space. */
int dab_get_pc_aggregates(dab_solver* s, int32_t* agg_of);

/* Test hook (no counterpart in the reference): the face-loop width of the cell-per-thread kernels this solver launches -- 6 when
 * every owned cell has exactly six faces (the unrolled NF=6 instantiations), 0 otherwise or with DAB_NOHEX6=1 at creation (the
 * rolled NF=0 loops). */
int dab_get_face_loop_width(dab_solver* s, int* nf);

/* Test hook (no counterpart in the reference): the transonic pressure equation of DATurboFoam (SIMPLE { transonic yes; }) at the
 * current state as the first SIMPLE iteration assembles it (momentum matrix and HbyA of the current U, rho = psi p) and one
 * BiCGStab solve of it from the current p; the states are not changed.  Rows: (diag[c] p_c + sum_k off[k*nC + c] p_nbr(k,c)) = b[c],
 * nbr[k*nC + c] the neighbour of the k-th face of cell c (-1 for boundary faces and unused slots).
 * coarse != 0 keeps the coarse space of the preconditioner; agg_of[c] is then the local aggregate of cell c (-1 without a coarse
 * space) and, if rc and yc are given, yc = Ac^-1 rc (n_agg entries) through the solver's coarse apply.  off == NULL: only *max_cf
 * and *n_agg are returned. */
int dab_transonic_pressure_probe(dab_solver* s, int coarse, int* max_cf, int* n_agg, int32_t* nbr, double* off, double* diag, double* b,
                                 double* x, int* iterations, int32_t* agg_of, const double* rc, double* yc);

/* calcPCMatWithFvMatrix(PCMat, turbOnly) (reference pyDASolvers.pyx:99-114 list, DASolver.C:2888-2988): the turbulence block of
 * the preconditioner taken from the relaxed nuTilda fvMatrix (diag / lower / upper, `div(pc)` convection, DASpalartAllmaras.C:
 * 490-529), scaled and transposed like the reference, as COO triplets (row, column, value) in the local state numbering -- what the
 * reference inserts into the PETSc Mat.  rows == NULL: only *nnz is returned.  turb_only == 0 is an error, as in the reference
 * (DAResidual::calcPCMatWithFvMatrix aborts for the SIMPLE solver family, DAResidual.C:295-300). */
int dab_calc_pc_mat_fvmatrix(dab_solver* s, int turb_only, int64_t* nnz, int32_t* rows, int32_t* cols, double* vals);

/* setSolverInput(inputName, inputType, inputSize, inputs, seeds): assign an input to the solver's fields before
 * solvePrimal / calcFunction (reference pyDASolvers.pyx:164-182, DASolver::setSolverInput -> DAInput::run;
 * DAInputPatchVelocity.C, DAInputStateVar.C).  Types: "patchVelocity" (|U|, angle of attack [deg]) and "stateVar".
 * `seeds` belongs to the reference's forward-mode AD and is ignored (may be NULL). */
int dab_set_solver_input(dab_solver* s, const char* input_name, const char* input_type, int input_size, const double* inputs,
                         const double* seeds);

/* solvePrimal(): SIMPLE iterations from the current states until the largest initial residual drops below
 * primalMinResTol or endTime is reached (reference pyDASolvers.pyx solvePrimal, DASimpleFoam.C:123-185,
 * DASolver.C:156-228).  *fail = 0/1 with the reference's checkPrimalFailure rule (residual misses the
 * tolerance by more than primalMinResTolDiff, or NaN).  The converged states are read with dab_get_of_fields. */
int dab_solve_primal(dab_solver* s, int* fail, dab_primal_stats* stats);

/* calcFunction(name) (reference DASolver.H calcFunction, DAFunctionForce.C:79-153) */
int dab_calc_function(dab_solver* s, const char* name, double* value);

/* getInputSize / getOutputSize (pyDASolvers.pyx:189-199) */
int dab_get_input_size(dab_solver* s, const char* name, const char* type, int64_t* out);
int dab_get_output_size(dab_solver* s, const char* name, const char* type, int64_t* out);

/* calcOutput(name, type, out) for type forceCouplingOutput (reference DAOutputForceCoupling.C:19-215): the wall force
 * Sf (p_b - pRef) + Sf & devRhoReff_b of every face of the output's patches split equally over the face's points;
 * out[3 * n + k] is component k on output node n.  The patches follow their names in sorted order; each patch lists
 * its points (this rank's faces only) in ascending label order, so a point shared by two patches appears once per
 * patch.  3 * nodes entries, possibly none. */
int dab_calc_output(dab_solver* s, const char* name, const char* type, double* out);

/* The global point index of every node of a forceCouplingOutput, in output order (dab_get_output_size / 3
 * entries).  On several ranks a point on a partition seam is a node of each rank that has faces around it. */
int dab_get_output_points(dab_solver* s, const char* name, int64_t* labels);

/* --- benchmarking hooks (no reference counterpart): run the product n times on device-resident
 * vectors and return the mean device time per launch sequence in milliseconds (CUDA events on the
 * solver's stream). which = 0: dRdWT*psi product (3 kernels), 1: R(W) (3 kernels),
 * 2/3/4: the reverse kernels RevA/RevB/RevC alone */
int dab_bench_device(dab_solver* s, int which, int n, double* ms_per_call, int64_t* kernel_launches);
/* upload the device-resident input vector used by dab_bench_device (untimed) */
int dab_bench_set_vector(dab_solver* s, const double* x);
/* algorithmic bytes of one dRdWT*psi product (DESIGN.md, SURVEY.md section 8d) */
int dab_algorithmic_bytes(dab_solver* s, int which, int64_t* bytes);

#ifdef __cplusplus
}
#endif
#endif
