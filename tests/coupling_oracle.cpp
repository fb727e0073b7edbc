// Test-only reference of forceCouplingOutput's face forces: the oracle (oracle/oracle.cpp, included whole and unchanged) plus the
// wall force vector of one boundary face, Sf (p_b - pRef) + Sf & devRhoReff_b (DAOutputForceCoupling.C:100-118), evaluated on the
// oracle's residual work arrays and taped against the states or the mesh points.  The arithmetic restates the face loop of the
// oracle's forceFunction (DAFunctionForce.C:79-153); tests/test_force_coupling.py checks it against orc_force / orc_dforce_dw.
// Built on first use by tests/coupling_oracle.py.
#include "../oracle/oracle.cpp"

namespace orc
{

template <class T>
V3<T> wallFaceForce(const Case& cs, const Geom<T>& g, const Work<T>& wk, int b, double pRef)
{
    const Topo& t = cs.t;
    const int nC = t.nC, f = t.nIF + b, c = t.own[f];
    V3<T> nh = (T(1.0) / g.magSf[f]) * g.Sf[f];
    T Gb[3][3];
    for (int j = 0; j < 3; j++)
    {
        T nG(0.0);
        for (int i = 0; i < 3; i++) nG += nh[i] * wk.gradU[((size_t)j * 3 + i) * nC + c];
        for (int i = 0; i < 3; i++) Gb[i][j] = wk.gradU[((size_t)j * 3 + i) * nC + c] + nh[i] * (wk.bU.sng[wk.bU.at(j, b)] - nG);
    }
    T tr = Gb[0][0] + Gb[1][1] + Gb[2][2];
    T nuEffB = cs.comp.on ? wk.muEB[b] : T(wk.bNut.val[b] + cs.par.nu); // compressible: devRhoReff = -rho*nuEff*dev(twoSymm(grad U))
    V3<T> F;
    for (int j = 0; j < 3; j++)
    {
        // (Sf & devRhoReff)_j = -nuEff * S_i * dev(twoSymm(G))_ij
        T s(0.0);
        for (int i = 0; i < 3; i++) s += g.Sf[f][i] * (Gb[i][j] + Gb[j][i]);
        s -= (2.0 / 3.0) * tr * g.Sf[f][j];
        F[j] = g.Sf[f][j] * (wk.bP.val[b] - pRef) - nuEffB * s;
    }
    return F;
}

// out[3 * b + k]: the wall force vectors of the faces of the patches in patchMask (bit p: patch p), zero on the other faces
template <class T>
void faceForces(const Case& cs, const Geom<T>& g, const std::vector<T>& W, unsigned patchMask, double pRef, std::vector<T>& out)
{
    std::vector<T> R;
    Work<T> wk;
    residual(cs, g, W, 0, R, &wk);
    const Topo& t = cs.t;
    out.assign((size_t)3 * t.nBF, T(0.0));
    for (int b = 0; b < t.nBF; b++)
        if ((patchMask >> t.bPatch[b]) & 1u)
        {
            const V3<T> ff = wallFaceForce(cs, g, wk, b, pRef);
            for (int k = 0; k < 3; k++) out[(size_t)3 * b + k] = ff[k];
        }
}

} // namespace orc

extern "C"
{

void cpl_face_forces(void* h, const double* W, unsigned patchMask, double pRef, double* out)
{
    Case* cs = (Case*)h;
    std::vector<double> w(W, W + cs->nDof()), F;
    faceForces<double>(*cs, cs->gd, w, patchMask, pRef, F);
    std::copy(F.begin(), F.end(), out);
}

// sum_b seeds[3b..3b+2] . F_b taped against the states (wrt 0: out[ndof], scaled like the reference if normalize) or the points
// (wrt 1: out[3 nP], through the geometry as orc_jtvec_xv)
void cpl_face_forces_jtvec(void* h, const double* W, unsigned patchMask, double pRef, const double* seeds, int wrt, int normalize, double* out)
{
    Case* cs = (Case*)h;
    Tape& tp = tape();
    tp.reset();
    const int n = cs->nDof(), nP = cs->t.nP;
    std::vector<AReal> w(n);
    std::vector<V3<AReal>> P(nP);
    std::vector<int> ids;
    for (int i = 0; i < n; i++)
    {
        w[i] = AReal(W[i]);
        if (wrt == 0)
        {
            w[i].registerInput();
            ids.push_back(w[i].id);
        }
    }
    for (int i = 0; i < nP; i++)
        for (int k = 0; k < 3; k++)
        {
            AReal a(cs->pts[3 * i + k]);
            if (wrt == 1)
            {
                a.registerInput();
                ids.push_back(a.id);
            }
            P[i][k] = a;
        }
    Geom<AReal> g;
    computeGeometry(cs->t, P, g);
    std::vector<AReal> F;
    faceForces<AReal>(*cs, g, w, patchMask, pRef, F);
    std::vector<double> adj(tp.size() + 1, 0.0);
    for (size_t i = 0; i < F.size(); i++)
        if (F[i].id) adj[F[i].id] += seeds[i];
    tp.evaluate(adj);
    for (size_t i = 0; i < ids.size(); i++) out[i] = adj[ids[i]];
    if (wrt == 0 && normalize) scaleStates(cs, out);
    tp.reset();
    cs->recorded = false;
}

} // extern "C"
