// C ABI of libdab200.so (include/dab200.h).  Compiled by nvcc as CUDA (`-x cu`, sm_90a).
#include "../../include/dab200.h"
#include "solver.hpp"
#include <cstring>
#include <string>

using namespace dab;

struct dab_solver
{
    Solver s;
};

static thread_local std::string g_err;
// communication callbacks for the next dab_create (test-only host build: torch.distributed/gloo drives the halos)
static dab_exchange_fn g_cbExchange = nullptr;
static dab_allreduce_fn g_cbAllreduce = nullptr;
static void* g_cbCtx = nullptr;

#define DAB_TRY try {
#define DAB_CATCH                                   \
    }                                               \
    catch (const std::exception& e)                 \
    {                                               \
        g_err = e.what();                           \
        return 1;                                   \
    }                                               \
    catch (...)                                     \
    {                                               \
        g_err = "unknown error";                    \
        return 1;                                   \
    }                                               \
    return 0;

static void need(const void* p, const char* what)
{
    if (!p) throw Error(std::string("null pointer: ") + what);
}
// every entry point that takes a solver makes the solver's device current first: another library (torch, a second engine handle)
// may have changed the calling thread's current device since dab_create (ADVICE round 1)
static void need(dab_solver* s, const char* what)
{
    if (!s) throw Error(std::string("null pointer: ") + what);
    s->s.be.makeCurrent();
}

extern "C"
{

const char* dab_last_error(void) { return g_err.c_str(); }

const char* dab_version(void)
{
#ifdef DAB_HOSTSIM
    return "dab200 0.1 (HOSTSIM test build -- not the product)";
#else
    return "dab200 0.1 (sm_90a)";
#endif
}

int dab_create(const char* case_dir, const char* args_all, const char* options_json, int device, int rank, int n_ranks,
               const void* nccl_unique_id, dab_solver** out)
{
    DAB_TRY
    need(case_dir, "case_dir");
    need(out, "out");
    dab_solver* h = new dab_solver();
    try
    {
        h->s.comm.cbExchange = g_cbExchange;
        h->s.comm.cbAllreduce = g_cbAllreduce;
        h->s.comm.cbCtx = g_cbCtx;
        h->s.create(case_dir, args_all ? args_all : "DASimpleFoam -python", options_json ? options_json : "", device, rank, n_ranks,
                    nccl_unique_id);
    }
    catch (...)
    {
        delete h;
        throw;
    }
    *out = h;
    DAB_CATCH
}

int dab_destroy(dab_solver* s)
{
    DAB_TRY
    if (s)
    {
        s->s.be.sync();
        s->s.comm.destroy();
        delete s;
    }
    DAB_CATCH
}

int dab_nccl_unique_id(void* out128)
{
    DAB_TRY
    need(out128, "out128");
#if !defined(DAB_HOSTSIM) && defined(DAB_WITH_NCCL)
    static_assert(sizeof(ncclUniqueId) == 128, "NCCL unique id size");
    ncclUniqueId id;
    NcclApi& N = NcclApi::get();
    ncclResult_t r = N.GetUniqueId(&id);
    if (r != ncclSuccess) throw Error(std::string("ncclGetUniqueId: ") + N.GetErrorString(r));
    memcpy(out128, &id, sizeof(id));
#else
    throw Error("NCCL is not built into this library");
#endif
    DAB_CATCH
}

int dab_n_local_adjoint_states(dab_solver* s, int64_t* out) { DAB_TRY need(s, "solver"); *out = s->s.nDof(); DAB_CATCH }
int dab_n_local_cells(dab_solver* s, int64_t* out) { DAB_TRY need(s, "solver"); *out = s->s.hm.nC; DAB_CATCH }
int dab_n_global_cells(dab_solver* s, int64_t* out) { DAB_TRY need(s, "solver"); *out = s->s.part.nGlobalCells; DAB_CATCH }
int dab_n_local_points(dab_solver* s, int64_t* out) { DAB_TRY need(s, "solver"); *out = s->s.hm.nP; DAB_CATCH }
int dab_volcoord_evaluations(dab_solver* s, int64_t* out) { DAB_TRY need(s, "solver"); *out = s->s.volc.nEval; DAB_CATCH }
int dab_n_local_faces(dab_solver* s, int64_t* out) { DAB_TRY need(s, "solver"); *out = s->s.hm.nF; DAB_CATCH }
int dab_n_local_internal_faces(dab_solver* s, int64_t* out) { DAB_TRY need(s, "solver"); *out = s->s.hm.nIF; DAB_CATCH }

int dab_update_options(dab_solver* s, const char* options_json)
{
    DAB_TRY
    need(s, "solver");
    s->s.applyOptions(options_json ? options_json : "", false);
    DAB_CATCH
}

int dab_update_of_fields(dab_solver* s, const double* states)
{
    DAB_TRY
    need(s, "solver");
    need(states, "states");
    s->s.updateOFFields(states);
    DAB_CATCH
}

int dab_get_of_fields(dab_solver* s, double* states)
{
    DAB_TRY
    need(s, "solver");
    need(states, "states");
    s->s.getOFFields(states);
    DAB_CATCH
}

int dab_get_of_mesh_points(dab_solver* s, double* points)
{
    DAB_TRY
    need(s, "solver");
    need(points, "points");
    memcpy(points, s->s.hm.points.data(), s->s.hm.points.size() * sizeof(double));
    DAB_CATCH
}

int dab_update_of_mesh(dab_solver* s, const double* points)
{
    DAB_TRY
    need(s, "solver");
    need(points, "points");
    s->s.updateMesh(points);
    DAB_CATCH
}

// OpenFOAM's time name of a value (general format, 6 significant digits: Time::timeName with the default precision)
static std::string timeNameOf(double t)
{
    char buf[64];
    snprintf(buf, sizeof buf, "%.6g", t);
    return buf;
}

int dab_write_adjoint_fields(dab_solver* s, const char* function, double write_time, const double* psi)
{
    DAB_TRY
    need(s, "solver");
    need(function, "function");
    need(psi, "psi");
    s->s.writeStateVector(timeNameOf(write_time), std::string("adjoint_") + function + "_", psi);
    DAB_CATCH
}

int dab_write_fields(dab_solver* s, double write_time)
{
    DAB_TRY
    need(s, "solver");
    std::vector<double> W(s->s.nDof());
    s->s.getOFFields(W.data());
    s->s.writeStateVector(timeNameOf(write_time), "", W.data());
    DAB_CATCH
}

int dab_check_mesh(dab_solver* s, double max_non_orth, double max_skewness, double max_aspect_ratio, int max_incorrectly_oriented_faces,
                   int* mesh_ok, double* report)
{
    DAB_TRY
    need(s, "solver");
    need(mesh_ok, "mesh_ok");
    const HostMesh::Quality q = s->s.hm.checkMesh(max_non_orth, max_skewness, max_aspect_ratio, max_incorrectly_oriented_faces);
    *mesh_ok = q.nFailedChecks == 0 ? 1 : 0;
    if (report)
    {
        const double r[DAB_CHECK_MESH_REPORT] = {q.maxNonOrth, q.avgNonOrth, q.maxSkewness, q.maxAspectRatio, q.minVolume, q.minFaceArea,
                                                 q.maxOpenness, (double)q.nSevereNonOrth, (double)q.nErrorNonOrth,
                                                 (double)q.nNegativePyramids, (double)q.nFailedChecks};
        for (int i = 0; i < DAB_CHECK_MESH_REPORT; i++) report[i] = r[i];
    }
    DAB_CATCH
}

int dab_read_state_vars(dab_solver* s, double time_val)
{
    DAB_TRY
    need(s, "solver");
    s->s.readStateVars(timeNameOf(time_val));
    DAB_CATCH
}

int dab_read_mesh_points(dab_solver* s, double time_val)
{
    DAB_TRY
    need(s, "solver");
    s->s.readMeshPoints(timeNameOf(time_val));
    DAB_CATCH
}

int dab_write_mesh_points(dab_solver* s, const double* points, const char* dir_name)
{
    DAB_TRY
    need(s, "solver");
    need(dir_name, "dir_name");
    s->s.writeMeshPoints(points ? points : s->s.hm.points.data(), dir_name);
    DAB_CATCH
}

int dab_write_sens_map_surface(dab_solver* s, const char* name, const double* dfdxs, const double* xs, int size, double time_name,
                               double* min_distance_norm)
{
    DAB_TRY
    need(s, "solver");
    need(name, "name");
    need(dfdxs, "dFdXs");
    need(xs, "Xs");
    const double nrm = s->s.writeSensMapSurface(name, dfdxs, xs, size, timeNameOf(time_name));
    if (min_distance_norm) *min_distance_norm = nrm;
    DAB_CATCH
}

int dab_write_sens_map_field(dab_solver* s, const char* name, const double* dfdfield, const char* field_type, double time_name)
{
    DAB_TRY
    need(s, "solver");
    need(name, "name");
    need(dfdfield, "dFdField");
    need(field_type, "field_type");
    const std::string ft(field_type);
    if (ft != "scalar" && ft != "vector") throw Error("writeSensMapField: fieldType can be either scalar or vector");
    s->s.writeSensMapField(name, dfdfield, ft == "vector", timeNameOf(time_name));
    DAB_CATCH
}

int dab_get_of_field(dab_solver* s, const char* name, const char* type, double* field)
{
    DAB_TRY
    need(s, "solver");
    need(name, "name");
    need(field, "field");
    (void)type;
    Solver& S = s->s;
    const std::string n(name);
    const size_t nC = S.hm.nC;
    if (n == "U") S.be.d2h(field, S.dU.p, 3 * nC * sizeof(double));
    else if (n == "p") S.be.d2h(field, S.dP.p, nC * sizeof(double));
    else if (n == "nuTilda") S.be.d2h(field, S.dNt.p, nC * sizeof(double));
    else if (n == "nut") { S.ensureRecorded(); S.be.d2h(field, S.rNut.p, nC * sizeof(double)); }
    else if (n == "yWall") memcpy(field, S.hm.yWall.data(), nC * sizeof(double));
    else if (n == "V") memcpy(field, S.hm.V.data(), nC * sizeof(double));
    else throw Error("getOFField: unknown field " + n);
    DAB_CATCH
}

int dab_get_residuals(dab_solver* s, int is_pc, double* residuals)
{
    DAB_TRY
    need(s, "solver");
    need(residuals, "residuals");
    s->s.getResiduals(is_pc, residuals);
    DAB_CATCH
}

int dab_calc_jac_t_vec_product(dab_solver* s, const char* input_name, const char* input_type, const double* input,
                               const char* output_name, const char* output_type, const double* seed, double* product)
{
    DAB_TRY
    need(s, "solver");
    need(input_type, "input_type");
    need(output_type, "output_type");
    need(seed, "seed");
    need(product, "product");
    (void)input_name;
    Solver& S = s->s;
    const std::string it(input_type), ot(output_type);
    if (it == "patchVelocity")
    {
        need(input_name, "input_name");
        need(input, "input");
        if (ot == "residual") S.patchVelocityProduct(input_name, input, seed, product);
        else if (ot == "function")
        {
            // only the flow-aligned direction modes (parallelToFlow / normalToFlow) depend on the angle of attack
            need(output_name, "output_name");
            S.setPatchVelocity(input_name, input);
            S.dFdPatchVelocity(output_name, seed[0], product);
        }
        else throw Error("calcJacTVecProduct: outputType " + ot + " is not supported");
        return 0;
    }
    if (it == "fvSourcePar")
    {
        need(input_name, "input_name");
        need(input, "input");
        if (ot == "residual") S.fvSourceParProduct(input_name, input, seed, nullptr, 1.0, product);
        else if (ot == "function")
        {
            need(output_name, "output_name");
            const std::string fn(output_name);
            S.fvSourceParProduct(input_name, input, nullptr, &fn, seed[0], product);
        }
        else throw Error("calcJacTVecProduct: outputType " + ot + " is not supported");
        return 0;
    }
    if (it == "patchVar")
    {
        need(input_name, "input_name");
        need(input, "input");
        if (ot == "residual") S.patchVarProduct(input_name, input, seed, nullptr, 1.0, product);
        else if (ot == "function")
        {
            need(output_name, "output_name");
            const std::string fn(output_name);
            S.patchVarProduct(input_name, input, nullptr, &fn, seed[0], product);
        }
        else throw Error("calcJacTVecProduct: outputType " + ot + " is not supported");
        return 0;
    }
    if (it == "volCoord")
    {
        // daInput->run: assign the point coordinates (DAInputVolCoord.C:35-70), then the transposed product
        if (input)
        {
            bool same = true;
            for (size_t i = 0; i < S.hm.points.size() && same; i++) same = (input[i] == S.hm.points[i]);
            if (!same) S.updateMesh(input);
        }
        if (ot == "residual") S.volCoordProduct(seed, {}, 1.0, product);
        else if (ot == "function")
        {
            need(output_name, "output_name");
            const FunctionDef& f = S.findFunction(output_name);
            S.ensureRecorded();
            S.volCoordProduct(nullptr, S.derivativeSpecs(f), seed[0], product); // at the unperturbed geometry
        }
        else if (ot == "forceCouplingOutput")
        {
            need(output_name, "output_name");
            S.forceCouplingdXv(output_name, seed, product);
        }
        else throw Error("calcJacTVecProduct: outputType " + ot + " is not supported");
        return 0;
    }
    if (it != "stateVar") throw Error("calcJacTVecProduct: inputType " + it + " is not supported (stateVar, patchVelocity, patchVar, volCoord)");
    // daInput->run(inputList): assign the input to the OpenFOAM fields (DAInputStateVar.C:35-140)
    if (input && !S.statesAreResident(input)) S.updateOFFields(input);
    if (ot == "residual") S.matVec(seed, product);
    else if (ot == "function")
    {
        need(output_name, "output_name");
        S.dFdW(output_name, seed[0], product);
    }
    else if (ot == "forceCouplingOutput")
    {
        need(output_name, "output_name");
        S.forceCouplingdW(output_name, seed, product);
    }
    else throw Error("calcJacTVecProduct: outputType " + ot + " is not supported (residual, function, forceCouplingOutput)");
    DAB_CATCH
}

int dab_drdwt_mat_vec(dab_solver* s, const double* x, double* y)
{
    DAB_TRY
    need(s, "solver");
    need(x, "x");
    need(y, "y");
    s->s.matVec(x, y);
    DAB_CATCH
}

int dab_calc_drdwt_pc(dab_solver* s)
{
    DAB_TRY
    need(s, "solver");
    s->s.calcPC();
    DAB_CATCH
}

int dab_set_comm_callbacks(dab_exchange_fn exchange, dab_allreduce_fn allreduce, void* ctx)
{
    DAB_TRY
#ifdef DAB_HOSTSIM
    g_cbExchange = exchange;
    g_cbAllreduce = allreduce;
    g_cbCtx = ctx;
#else
    (void)exchange; (void)allreduce; (void)ctx;
    throw Error("communication callbacks exist only in the test build; the product uses NCCL");
#endif
    DAB_CATCH
}

int dab_get_local_to_global(dab_solver* s, int what, int64_t* out)
{
    DAB_TRY
    need(s, "solver");
    need(out, "out");
    Solver& S = s->s;
    if (what == 0)
        for (int c = 0; c < S.hm.nC; c++) out[c] = S.partitioned ? S.part.cellGlobal[c] : c;
    else if (what == 1)
        for (int f = 0; f < S.hm.nF; f++) out[f] = S.partitioned ? S.part.faceGlobal[f] : f;
    else if (what == 2)
        for (int f = 0; f < S.hm.nF; f++) out[f] = S.partitioned ? S.part.faceOwned[f] : 1;
    else throw Error("dab_get_local_to_global: what must be 0 (cells), 1 (faces) or 2 (face ownership)");
    DAB_CATCH
}

int dab_get_pc_matrix(dab_solver* s, int64_t* n_rows, int64_t* nnz, int64_t* row_ptr, int32_t* cols, double* vals)
{
    DAB_TRY
    need(s, "solver");
    need(n_rows, "n_rows");
    need(nnz, "nnz");
    Solver& S = s->s;
    if (!row_ptr)
    {
        *n_rows = S.kry.n;
        *nnz = S.kry.nnz;
        return 0;
    }
    need(cols, "cols");
    need(vals, "vals");
    std::vector<int64_t> rp;
    std::vector<int32_t> cl;
    std::vector<double> vl;
    S.exportPC(rp, cl, vl);
    if ((int64_t)cl.size() > *nnz || (int64_t)rp.size() - 1 > *n_rows) throw Error("dab_get_pc_matrix: the buffers are too small");
    *n_rows = (int64_t)rp.size() - 1;
    *nnz = (int64_t)cl.size();
    std::copy(rp.begin(), rp.end(), row_ptr);
    std::copy(cl.begin(), cl.end(), cols);
    std::copy(vl.begin(), vl.end(), vals);
    DAB_CATCH
}

int dab_get_pc_factors(dab_solver* s, int64_t* n_rows, int64_t* nnz, int64_t* row_ptr, int32_t* cols, double* vals, int32_t* perm,
                       int32_t* colour)
{
    DAB_TRY
    need(s, "solver");
    need(n_rows, "n_rows");
    need(nnz, "nnz");
    Solver& S = s->s;
    if (!S.kry.pcFactored) throw Error("dab_get_pc_factors: no ILU(0) factorisation: call dab_calc_drdwt_pc first");
    if (!row_ptr)
    {
        *n_rows = S.kry.n;
        *nnz = S.kry.nnz;
        return 0;
    }
    need(cols, "cols");
    need(vals, "vals");
    need(perm, "perm");
    need(colour, "colour");
    std::vector<int64_t> rp;
    std::vector<int32_t> cl, pm, co;
    std::vector<double> vl;
    S.exportPCFactors(rp, cl, vl, pm, co);
    if ((int64_t)cl.size() > *nnz || (int64_t)rp.size() - 1 > *n_rows) throw Error("dab_get_pc_factors: the buffers are too small");
    *n_rows = (int64_t)rp.size() - 1;
    *nnz = (int64_t)cl.size();
    std::copy(rp.begin(), rp.end(), row_ptr);
    std::copy(cl.begin(), cl.end(), cols);
    std::copy(vl.begin(), vl.end(), vals);
    std::copy(pm.begin(), pm.end(), perm);
    std::copy(co.begin(), co.end(), colour);
    DAB_CATCH
}

int dab_get_pc_aggregates(dab_solver* s, int32_t* agg_of)
{
    DAB_TRY
    need(s, "solver");
    need(agg_of, "agg_of");
    Solver& S = s->s;
    const Coarse& Cs = S.kry.coarse;
    if (!Cs.enabled || !Cs.valid) throw Error("dab_get_pc_aggregates: the preconditioner has no coarse space (adjEqnOption.coarseAggregates)");
    std::vector<int32_t> a((size_t)S.hm.nC);
    S.be.d2h(a.data(), Cs.dAggOf.p, a.size() * sizeof(int32_t));
    for (int c = 0; c < S.hm.nC; c++) agg_of[c] = Cs.aggBase + a[c];
    DAB_CATCH
}

int dab_get_face_loop_width(dab_solver* s, int* nf)
{
    DAB_TRY
    need(s, "solver");
    need(nf, "nf");
    *nf = s->s.hex6 ? 6 : 0;
    DAB_CATCH
}

int dab_transonic_pressure_probe(dab_solver* s, int coarse, int* max_cf, int* n_agg, int32_t* nbr, double* off, double* diag, double* b,
                                 double* x, int* iterations, int32_t* agg_of, const double* rc, double* yc)
{
    DAB_TRY
    need(s, "solver");
    need(max_cf, "max_cf");
    need(n_agg, "n_agg");
    Solver& S = s->s;
    S.primalSetup();
    *max_cf = S.hm.maxCF;
    *n_agg = S.primal.nAgg;
    if (!off) return 0;
    need(nbr, "nbr");
    need(diag, "diag");
    need(b, "b");
    need(x, "x");
    need(iterations, "iterations");
    need(agg_of, "agg_of");
    std::vector<double> o, d, bb, xx;
    std::vector<int32_t> a;
    S.transonicPressureProbe(coarse, o, d, bb, xx, *iterations, a, rc, yc);
    const size_t nC = (size_t)S.hm.nC;
    for (size_t i = 0; i < (size_t)S.hm.maxCF * nC; i++) nbr[i] = S.hm.cellNbr[i] < (int)nC ? S.hm.cellNbr[i] : -1;
    std::copy(o.begin(), o.end(), off);
    std::copy(d.begin(), d.end(), diag);
    std::copy(bb.begin(), bb.end(), b);
    std::copy(xx.begin(), xx.end(), x);
    std::copy(a.begin(), a.end(), agg_of);
    DAB_CATCH
}

int dab_calc_pc_mat_fvmatrix(dab_solver* s, int turb_only, int64_t* nnz, int32_t* rows, int32_t* cols, double* vals)
{
    DAB_TRY
    need(s, "solver");
    need(nnz, "nnz");
    std::vector<int32_t> r, c;
    std::vector<double> v;
    s->s.calcPCMatWithFvMatrix(turb_only, r, c, v);
    if (!rows)
    {
        *nnz = (int64_t)v.size();
        return 0;
    }
    need(cols, "cols");
    need(vals, "vals");
    if ((int64_t)v.size() > *nnz) throw Error("dab_calc_pc_mat_fvmatrix: the buffers are too small");
    *nnz = (int64_t)v.size();
    std::copy(r.begin(), r.end(), rows);
    std::copy(c.begin(), c.end(), cols);
    std::copy(v.begin(), v.end(), vals);
    DAB_CATCH
}

int dab_pc_apply(dab_solver* s, const double* v, double* z)
{
    DAB_TRY
    need(s, "solver");
    need(v, "v");
    need(z, "z");
    Solver& S = s->s;
    if (!S.kry.pcValid) S.calcPC();
    S.be.h2d(S.dX.p, v, (size_t)S.nDof() * sizeof(double));
    S.applyPC(S.dX.p, S.dY2.p);
    S.be.d2h(z, S.dY2.p, (size_t)S.nDof() * sizeof(double));
    DAB_CATCH
}

int dab_set_solver_input(dab_solver* s, const char* input_name, const char* input_type, int input_size, const double* inputs,
                         const double* seeds)
{
    DAB_TRY
    need(s, "solver");
    need(input_type, "input_type");
    need(inputs, "inputs");
    (void)seeds;
    Solver& S = s->s;
    const std::string it(input_type);
    if (it == "patchVelocity")
    {
        need(input_name, "input_name");
        if (input_size != 2) throw Error("setSolverInput: patchVelocity takes 2 values (|U|, angle of attack)");
        S.setPatchVelocity(input_name, inputs);
    }
    else if (it == "stateVar")
    {
        if (input_size != S.nDof()) throw Error("setSolverInput: stateVar has the wrong size");
        S.updateOFFields(inputs);
    }
    else if (it == "volCoord")
    {
        if ((size_t)input_size != S.hm.points.size()) throw Error("setSolverInput: volCoord has the wrong size");
        S.updateMesh(inputs);
    }
    else if (it == "fvSourcePar")
    {
        need(input_name, "input_name");
        if ((size_t)input_size != S.findFvSourcePar(input_name).indices.size()) throw Error("setSolverInput: fvSourcePar has the wrong size");
        S.setFvSourcePar(input_name, inputs);
    }
    else if (it == "patchVar")
    {
        need(input_name, "input_name");
        if (input_size != S.findPatchVar(input_name).nComp) throw Error("setSolverInput: patchVar has the wrong size");
        S.setPatchVar(input_name, inputs);
    }
    else
        throw Error("setSolverInput: inputType " + it + " is not supported (patchVelocity, patchVar, stateVar, volCoord)");
    DAB_CATCH
}

int dab_solve_primal(dab_solver* s, int* fail, dab_primal_stats* stats)
{
    DAB_TRY
    need(s, "solver");
    PrimalStats st;
    const int f = s->s.solvePrimal(st);
    if (fail) *fail = f;
    if (stats)
    {
        stats->iterations = st.iterations;
        stats->converged = st.converged;
        stats->p_iterations = st.pIterations;
        stats->reserved = 0;
        stats->max_residual = st.maxRes;
        for (int j = 0; j < 3; j++) stats->res_u[j] = st.resU[j];
        stats->res_p = st.resP;
        stats->res_nutilda = st.resN;
        stats->seconds = st.sec;
    }
    DAB_CATCH
}

int dab_run_fp_adj(dab_solver* s, const double* dfdw, double* psi, int* fail, dab_ksp_stats* stats)
{
    DAB_TRY
    need(s, "solver");
    need(dfdw, "dFdW");
    need(psi, "psi");
    KspStats st;
    const int f = s->s.solveFixedPoint(dfdw, psi, st);
    if (fail) *fail = f;
    if (stats)
    {
        stats->iterations = st.iterations;
        stats->converged_reason = st.reason;
        stats->initial_residual = st.r0;
        stats->final_residual = st.rn;
        stats->solve_seconds = st.solveSec;
        stats->pc_setup_seconds = st.pcSec;
        stats->pc_assemblies = s->s.kry.pcAssemblies;
        stats->n_matvec = st.nMatvec;
    }
    DAB_CATCH
}

int dab_solve_linear_eqn(dab_solver* s, const double* rhs, double* sol, int* fail, dab_ksp_stats* stats)
{
    DAB_TRY
    need(s, "solver");
    need(rhs, "rhs");
    need(sol, "sol");
    KspStats st;
    const int f = s->s.solveLinearEqn(rhs, sol, st);
    if (fail) *fail = f;
    if (stats)
    {
        stats->iterations = st.iterations;
        stats->converged_reason = st.reason;
        stats->initial_residual = st.r0;
        stats->final_residual = st.rn;
        stats->solve_seconds = st.solveSec;
        stats->pc_setup_seconds = st.pcSec;
        stats->pc_assemblies = s->s.kry.pcAssemblies;
        stats->n_matvec = st.nMatvec;
    }
    DAB_CATCH
}

int dab_calc_function(dab_solver* s, const char* name, double* value)
{
    DAB_TRY
    need(s, "solver");
    need(name, "name");
    need(value, "value");
    *value = s->s.calcFunction(name);
    DAB_CATCH
}

int dab_get_input_size(dab_solver* s, const char* name, const char* type, int64_t* out)
{
    DAB_TRY
    need(s, "solver");
    need(type, "type");
    (void)name;
    if (std::string(type) == "stateVar") *out = s->s.nDof();
    else if (std::string(type) == "patchVelocity") *out = 2;
    else if (std::string(type) == "volCoord") *out = (int64_t)s->s.hm.points.size();
    else if (std::string(type) == "patchVar") { need(name, "name"); *out = s->s.findPatchVar(name).nComp; }
    else if (std::string(type) == "fvSourcePar") { need(name, "name"); *out = (int64_t)s->s.findFvSourcePar(name).indices.size(); }
    else throw Error(std::string("getInputSize: unsupported input type ") + type);
    DAB_CATCH
}

int dab_get_output_size(dab_solver* s, const char* name, const char* type, int64_t* out)
{
    DAB_TRY
    need(s, "solver");
    need(type, "type");
    const std::string t(type);
    if (t == "residual") *out = s->s.nDof();
    else if (t == "function") *out = 1;
    else if (t == "forceCouplingOutput")
    {
        need(name, "name");
        *out = s->s.couplingSize(name);
    }
    else throw Error("getOutputSize: unsupported output type " + t);
    DAB_CATCH
}

int dab_calc_output(dab_solver* s, const char* name, const char* type, double* out)
{
    DAB_TRY
    need(s, "solver");
    need(name, "name");
    need(type, "type");
    need(out, "out");
    const std::string t(type);
    if (t != "forceCouplingOutput") throw Error("calcOutput: output type " + t + " is not supported (forceCouplingOutput)");
    s->s.calcForceCoupling(name, out);
    DAB_CATCH
}

int dab_get_output_points(dab_solver* s, const char* name, int64_t* labels)
{
    DAB_TRY
    need(s, "solver");
    need(name, "name");
    need(labels, "labels");
    const std::vector<int64_t>& n = s->s.findForceCoupling(name).nodes;
    std::copy(n.begin(), n.end(), labels);
    DAB_CATCH
}

int dab_bench_set_vector(dab_solver* s, const double* x)
{
    DAB_TRY
    need(s, "solver");
    need(x, "x");
    s->s.be.h2d(s->s.dX.p, x, (size_t)s->s.nDof() * sizeof(double));
    DAB_CATCH
}

int dab_bench_device(dab_solver* s, int which, int n, double* ms_per_call, int64_t* kernel_launches)
{
    DAB_TRY
    need(s, "solver");
    need(ms_per_call, "ms_per_call");
    Solver& S = s->s;
    S.ensureRecorded();
    const long l0 = S.be.launches;
    auto t = S.be.timer();
    S.be.sync();
    t.start();
    for (int i = 0; i < n; i++)
    {
        switch (which)
        {
        case 0: S.matVecDev(S.dX.p, S.dY2.p); break;
        case 1: S.forward(0, S.dR.p); break;
        case 2: S.benchKernel(0); break;
        case 3: S.benchKernel(1); break;
        case 4: S.benchKernel(2); break;
        default: throw Error("dab_bench_device: unknown selector");
        }
    }
    *ms_per_call = t.stopMs() / (n > 0 ? n : 1);
    if (kernel_launches) *kernel_launches = S.be.launches - l0;
    DAB_CATCH
}

int dab_algorithmic_bytes(dab_solver* s, int which, int64_t* bytes)
{
    DAB_TRY
    need(s, "solver");
    need(bytes, "bytes");
    const HostMesh& m = s->s.hm;
    const int64_t nDof = s->s.nDof();
    // SURVEY.md section 8d: W, psi, y (or W, R) + face geometry/addressing + cell geometry, each read once
    const int64_t vecs = which == 0 ? 3 : 2;
    *bytes = 8 * vecs * nDof + (int64_t)m.nIF * (8 * 10 + 4 * 2) + (int64_t)m.nBF * (8 * 6 + 4 * 2) + (int64_t)m.nC * (8 * 5);
    DAB_CATCH
}

} // extern "C"
