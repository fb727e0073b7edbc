"""Synthetic OpenFOAM cases for the adjoint hot path.

The reference ships no mesh: every test `chdir`s into a case directory that is downloaded at test
time (reference tests/Allrun:9-18).  This module generates cases of the same *shape* as the ones
the reference's tests and BASELINE.json name -- a one-cell-thick NACA0012 O-grid with patches
`wing` (wall), `inout` (farfield) and two `symmetry` planes (reference
tests/runRegTests_AeroOpt.py:29-101), optionally extruded to a 3-D wing, and a convergent channel
(reference tests/runRegTests_DASimpleFoamForward.py:32) -- and writes them in OpenFOAM `polyMesh`
format (ASCII, or the `format binary` variant for million-cell meshes) together with `0/`,
`constant/` and `system/` dictionaries that the C++ host reader of the engine parses.

It is input synthesis only: nothing here is on the timed path.
"""
from __future__ import annotations

import os
import numpy as np

# ----------------------------------------------------------------------------------------------
# mesh container
# ----------------------------------------------------------------------------------------------


class PolyMesh:
    """points (nP,3) f64; faces (nF,4) i32 (quads; triangles are padded with -1 in the last column);
    owner (nF) i32; neighbour (nIF) i32; patches: list of dict(name,type,start,size).  Internal faces
    come first, ordered by (owner, neighbour); boundary faces are grouped patch by patch (OpenFOAM
    convention)."""

    def __init__(self, points, faces, owner, neighbour, patches):
        self.points = np.ascontiguousarray(points, dtype=np.float64)
        self.faces = np.ascontiguousarray(faces, dtype=np.int32)
        self.owner = np.ascontiguousarray(owner, dtype=np.int32)
        self.neighbour = np.ascontiguousarray(neighbour, dtype=np.int32)
        self.patches = patches

    @property
    def n_cells(self):
        return int(self.owner.max()) + 1

    @property
    def n_faces(self):
        return self.faces.shape[0]

    @property
    def n_internal_faces(self):
        return self.neighbour.shape[0]

    @property
    def n_points(self):
        return self.points.shape[0]

    @property
    def face_sizes(self):
        return (self.faces >= 0).sum(axis=1).astype(np.int32)

    def face_offsets_labels(self):
        """CSR (offsets, labels) of the face -> point lists."""
        sz = self.face_sizes
        off = np.concatenate([[0], np.cumsum(sz)]).astype(np.int32)
        lab = self.faces[self.faces >= 0].astype(np.int32)
        return off, lab


def _naca0012_y(x):
    # closed trailing edge variant (last coefficient -0.1036)
    return 0.6 * (0.2969 * np.sqrt(np.maximum(x, 0.0)) - 0.1260 * x - 0.3516 * x**2 + 0.2843 * x**3 - 0.1036 * x**4)


def _assemble(points, quads, cell_a, cell_b, patch_of_bface, patch_defs, cell_centres, family_major=None, bface_by_owner=False):
    """Orient faces (normal owner->neighbour / outward), sort, and build a PolyMesh.

    quads: (n,4) point ids; cell_a: (n,) one adjacent cell; cell_b: (n,) other cell or -1;
    patch_of_bface: (n,) patch index for boundary faces (ignored for internal)."""
    quads = quads.copy()
    internal = cell_b >= 0
    own = np.where(internal, np.minimum(cell_a, cell_b), cell_a)
    nei = np.where(internal, np.maximum(cell_a, cell_b), -1)
    tri = quads[:, 3] < 0
    qq = quads.copy()
    qq[tri, 3] = qq[tri, 0]  # a triangle as a degenerate quad: same area vector, centre slightly off (only used for orientation)
    p = points[qq]  # (n,4,3)
    fc = p.mean(axis=1)
    # area vector of a quad by its diagonals
    nrm = 0.5 * np.cross(p[:, 2] - p[:, 0], p[:, 3] - p[:, 1])
    ref = np.where(internal[:, None], cell_centres[np.maximum(nei, 0)] - cell_centres[own], fc - cell_centres[own])
    flip = np.einsum("ij,ij->i", nrm, ref) < 0
    fq = flip & ~tri
    quads[fq] = quads[fq][:, ::-1]
    ft = flip & tri
    quads[ft, :3] = quads[ft, :3][:, ::-1]
    # internal faces sorted by (owner, neighbour)
    ii = np.nonzero(internal)[0]
    if family_major is not None:
        # keep the generation order of the face families (all i-faces, then j-faces, then k-faces), each sorted by owner:
        # faces that sit in the same slot of consecutive cells are then consecutive in memory
        fam = np.asarray(family_major)[ii]
        order_i = ii[np.lexsort((own[ii], fam))]
    else:
        order_i = ii[np.lexsort((nei[ii], own[ii]))]
    bi = np.nonzero(~internal)[0]
    # boundary faces patch by patch, inside a patch by owner cell (the order OpenFOAM's renumberMesh leaves): the boundary
    # faces of consecutive cells are consecutive in memory
    order_b = bi[np.lexsort((own[bi], patch_of_bface[bi]))] if bface_by_owner else bi[np.lexsort((np.arange(bi.size), patch_of_bface[bi]))]
    order = np.concatenate([order_i, order_b])
    faces = quads[order]
    owner = own[order]
    neighbour = nei[order_i]
    patches = []
    start = order_i.size
    pb = patch_of_bface[order_b]
    for k, (name, typ) in enumerate(patch_defs):
        n = int(np.count_nonzero(pb == k))
        patches.append(dict(name=name, type=typ, start=start, size=n))
        start += n
    return PolyMesh(points, faces, owner, neighbour, patches)


def naca0012_ogrid(ni=100, nj=50, nk=1, radius=20.0, span=0.1, first_dy=2.0e-3, tile=None, family_major=False, bface_by_owner=None,
                   sweep=0.0, taper=1.0):
    """NACA0012 O-grid: ni cells around the airfoil, nj cells radially (geometric stretching
    from `first_dy` chord at the wall to the farfield circle of `radius` chords), nk cells in z.
    Patches: wing (wall), inout (patch), sym1/sym2 (symmetry).
    sweep / taper (nk > 1): a swept, tapered wing between the two symmetry planes -- the section at span station z is the root
    section scaled about its leading edge by 1 + (taper - 1) z/span and shifted downstream by sweep*z (fully 3-D hexahedra:
    no face is aligned with a coordinate plane except the symmetry planes).  tile may be (ti, tj) or (ti, tj, tk)."""
    assert ni % 2 == 0
    th = 2.0 * np.pi * np.arange(ni) / ni
    xa = 0.5 * (1.0 + np.cos(th))
    ya = np.where(th <= np.pi, 1.0, -1.0) * _naca0012_y(xa)
    # farfield circle around mid-chord
    xf = 0.5 + radius * np.cos(th)
    yf = radius * np.sin(th)
    # radial distribution s_j in [0,1], geometric growth
    n = nj
    lo, hi = 1.0 + 1e-9, 2.0
    tot = radius

    def total(r):
        e = n * np.log(r)
        if e > 700.0:  # r**n would overflow (thousands of radial cells): certainly beyond the target length
            return np.inf
        return first_dy * np.expm1(e) / (r - 1.0)

    for _ in range(200):
        mid = 0.5 * (lo + hi)
        if total(mid) > tot:
            hi = mid
        else:
            lo = mid
    r = 0.5 * (lo + hi)
    s = np.concatenate([[0.0], np.cumsum(first_dy * r ** np.arange(n))])
    s = s / s[-1]
    X = xa[None, :] + s[:, None] * (xf - xa)[None, :]  # (nj+1, ni)
    Y = ya[None, :] + s[:, None] * (yf - ya)[None, :]
    z = np.linspace(0.0, span, nk + 1)
    npl = ni * (nj + 1)
    points = np.empty(((nk + 1) * npl, 3))
    for k in range(nk + 1):
        sc = 1.0 + (taper - 1.0) * z[k] / span
        # the far field stays the root's circle: only the near-wall part of the grid follows the local chord
        blend = (1.0 - s)[:, None] if (taper != 1.0 or sweep != 0.0) else 0.0
        points[k * npl:(k + 1) * npl, 0] = (X + blend * ((sc - 1.0) * X + sweep * z[k])).ravel()
        points[k * npl:(k + 1) * npl, 1] = (Y + blend * (sc - 1.0) * Y).ravel()
        points[k * npl:(k + 1) * npl, 2] = z[k]

    def pid(i, j, k):
        return (i % ni) + ni * (j + (nj + 1) * k)

    def cid_lex(i, j, k):
        return (i % ni) + ni * (j + nj * k)

    if tile is None:
        cid = cid_lex
    else:
        # tile-major cell numbering (ti x tj cells per tile): neighbouring cells get nearby indices in both directions
        ti, tj = tile[0], tile[1]
        tk = tile[2] if len(tile) > 2 else 1
        nti, ntj = (ni + ti - 1) // ti, (nj + tj - 1) // tj
        if tk <= 1:
            ii, jj = np.meshgrid(np.arange(ni), np.arange(nj), indexing="ij")
            key = ((jj // tj) * nti + (ii // ti)) * (ti * tj) + (jj % tj) * ti + (ii % ti)
            order = np.argsort(key.ravel(), kind="stable")  # positions in lexicographic (i,j) raveled as i*nj + j
            rank2d = np.empty(ni * nj, dtype=np.int64)
            rank2d[order] = np.arange(ni * nj)
            rank2d = rank2d.reshape(ni, nj)

            def cid(i, j, k):
                return rank2d[i % ni, j] + ni * nj * k
        else:
            # 3-D bricks of ti x tj x tk cells, numbered brick by brick, i fastest inside a brick
            ii, jj, kk = np.meshgrid(np.arange(ni), np.arange(nj), np.arange(nk), indexing="ij")
            key = (((kk // tk) * ntj + (jj // tj)) * nti + (ii // ti)) * (ti * tj * tk) + ((kk % tk) * tj + (jj % tj)) * ti + (ii % ti)
            order = np.argsort(key.ravel(), kind="stable")
            rank3d = np.empty(ni * nj * nk, dtype=np.int64)
            rank3d[order] = np.arange(ni * nj * nk)
            rank3d = rank3d.reshape(ni, nj, nk)

            def cid(i, j, k):
                return rank3d[i % ni, j, k]

    I, J, K = np.meshgrid(np.arange(ni), np.arange(nj), np.arange(nk), indexing="ij")
    I, J, K = I.ravel(), J.ravel(), K.ravel()
    # cell centres (mean of 8 corners) for orientation
    corners = [pid(I + a, J + b, K + c) for a in (0, 1) for b in (0, 1) for c in (0, 1)]
    cc = np.zeros((ni * nj * nk, 3))
    cells = cid(I, J, K)
    acc = sum(points[c] for c in corners) / 8.0
    cc[cells] = acc

    quads, ca, cb, pf = [], [], [], []

    def add(q, a, b, patch):
        quads.append(np.stack(q, axis=1))
        ca.append(a)
        cb.append(b)
        pf.append(np.full(a.shape, patch, dtype=np.int64))

    # i-faces (periodic in i): between (i,j,k) and (i+1,j,k)
    add([pid(I + 1, J, K), pid(I + 1, J + 1, K), pid(I + 1, J + 1, K + 1), pid(I + 1, J, K + 1)],
        cid(I, J, K), cid(I + 1, J, K), -1)
    # j-faces
    m = J >= 1
    add([pid(I[m], J[m], K[m]), pid(I[m] + 1, J[m], K[m]), pid(I[m] + 1, J[m], K[m] + 1), pid(I[m], J[m], K[m] + 1)],
        cid(I[m], J[m] - 1, K[m]), cid(I[m], J[m], K[m]), -1)
    # k-faces
    m = K >= 1
    if m.any():
        add([pid(I[m], J[m], K[m]), pid(I[m] + 1, J[m], K[m]), pid(I[m] + 1, J[m] + 1, K[m]), pid(I[m], J[m] + 1, K[m])],
            cid(I[m], J[m], K[m] - 1), cid(I[m], J[m], K[m]), -1)
    # boundary: wing (j=0), inout (j=nj), sym1 (k=0), sym2 (k=nk)
    m = J == 0
    add([pid(I[m], 0 * J[m], K[m]), pid(I[m] + 1, 0 * J[m], K[m]), pid(I[m] + 1, 0 * J[m], K[m] + 1), pid(I[m], 0 * J[m], K[m] + 1)],
        cid(I[m], J[m], K[m]), np.full(m.sum(), -1), 0)
    m = J == nj - 1
    add([pid(I[m], J[m] + 1, K[m]), pid(I[m] + 1, J[m] + 1, K[m]), pid(I[m] + 1, J[m] + 1, K[m] + 1), pid(I[m], J[m] + 1, K[m] + 1)],
        cid(I[m], J[m], K[m]), np.full(m.sum(), -1), 1)
    m = K == 0
    add([pid(I[m], J[m], K[m]), pid(I[m] + 1, J[m], K[m]), pid(I[m] + 1, J[m] + 1, K[m]), pid(I[m], J[m] + 1, K[m])],
        cid(I[m], J[m], K[m]), np.full(m.sum(), -1), 2)
    m = K == nk - 1
    add([pid(I[m], J[m], K[m] + 1), pid(I[m] + 1, J[m], K[m] + 1), pid(I[m] + 1, J[m] + 1, K[m] + 1), pid(I[m], J[m] + 1, K[m] + 1)],
        cid(I[m], J[m], K[m]), np.full(m.sum(), -1), 3)

    quads_list = quads
    quads = np.concatenate(quads).astype(np.int32)
    ca = np.concatenate(ca).astype(np.int64)
    cb = np.concatenate(cb).astype(np.int64)
    pf = np.concatenate(pf)
    defs = [("wing", "wall"), ("inout", "patch"), ("sym1", "symmetry"), ("sym2", "symmetry")]
    fam = np.concatenate([np.full(q.shape[0], i) for i, q in enumerate(quads_list)]) if family_major else None
    # tile-major cell numbering comes with boundary faces ordered by owner cell (the order OpenFOAM's renumberMesh leaves)
    return _assemble(points, quads, ca, cb, pf, defs, cc, family_major=fam,
                     bface_by_owner=(tile is not None) if bface_by_owner is None else bface_by_owner)


def channel(nx=20, ny=10, nz=1, lx=2.0, ly=0.5, lz=0.1, contraction=0.3, skew=0.15):
    """Convergent channel: inlet (x=0), outlet (x=lx), lower/upper walls, two symmetry planes.
    The upper wall descends by `contraction`*ly and interior lines are sheared by `skew`
    so the mesh is non-orthogonal (exercises the corrected snGrad / laplacian terms)."""
    xs = np.linspace(0.0, lx, nx + 1)
    et = np.linspace(0.0, 1.0, ny + 1)
    zs = np.linspace(0.0, lz, nz + 1)
    h = ly * (1.0 - contraction * 0.5 * (1.0 - np.cos(np.pi * xs / lx)))
    Xg = xs[:, None] + skew * ly * np.sin(np.pi * et)[None, :] * np.sin(np.pi * xs / lx)[:, None]
    Yg = et[None, :] * h[:, None]

    def pid(i, j, k):
        return i + (nx + 1) * (j + (ny + 1) * k)

    def cid(i, j, k):
        return i + nx * (j + ny * k)

    points = np.empty(((nx + 1) * (ny + 1) * (nz + 1), 3))
    Ip, Jp, Kp = np.meshgrid(np.arange(nx + 1), np.arange(ny + 1), np.arange(nz + 1), indexing="ij")
    idx = pid(Ip, Jp, Kp).ravel()
    points[idx, 0] = Xg[Ip.ravel(), Jp.ravel()]
    points[idx, 1] = Yg[Ip.ravel(), Jp.ravel()]
    points[idx, 2] = zs[Kp.ravel()]

    I, J, K = np.meshgrid(np.arange(nx), np.arange(ny), np.arange(nz), indexing="ij")
    I, J, K = I.ravel(), J.ravel(), K.ravel()
    corners = [pid(I + a, J + b, K + c) for a in (0, 1) for b in (0, 1) for c in (0, 1)]
    cc = np.zeros((nx * ny * nz, 3))
    cc[cid(I, J, K)] = sum(points[c] for c in corners) / 8.0

    quads, ca, cb, pf = [], [], [], []

    def add(q, a, b, patch):
        quads.append(np.stack(q, axis=1))
        ca.append(a)
        cb.append(b)
        pf.append(np.full(a.shape, patch, dtype=np.int64))

    def xface(i, j, k):
        return [pid(i, j, k), pid(i, j + 1, k), pid(i, j + 1, k + 1), pid(i, j, k + 1)]

    def yface(i, j, k):
        return [pid(i, j, k), pid(i + 1, j, k), pid(i + 1, j, k + 1), pid(i, j, k + 1)]

    def zface(i, j, k):
        return [pid(i, j, k), pid(i + 1, j, k), pid(i + 1, j + 1, k), pid(i, j + 1, k)]

    m = I >= 1
    add(xface(I[m], J[m], K[m]), cid(I[m] - 1, J[m], K[m]), cid(I[m], J[m], K[m]), -1)
    m = J >= 1
    add(yface(I[m], J[m], K[m]), cid(I[m], J[m] - 1, K[m]), cid(I[m], J[m], K[m]), -1)
    m = K >= 1
    if m.any():
        add(zface(I[m], J[m], K[m]), cid(I[m], J[m], K[m] - 1), cid(I[m], J[m], K[m]), -1)
    none = lambda m: np.full(int(m.sum()), -1)
    m = I == 0
    add(xface(I[m], J[m], K[m]), cid(I[m], J[m], K[m]), none(m), 0)
    m = I == nx - 1
    add(xface(I[m] + 1, J[m], K[m]), cid(I[m], J[m], K[m]), none(m), 1)
    m = J == 0
    add(yface(I[m], J[m], K[m]), cid(I[m], J[m], K[m]), none(m), 2)
    m = J == ny - 1
    add(yface(I[m], J[m] + 1, K[m]), cid(I[m], J[m], K[m]), none(m), 2)
    m = K == 0
    add(zface(I[m], J[m], K[m]), cid(I[m], J[m], K[m]), none(m), 3)
    m = K == nz - 1
    add(zface(I[m], J[m], K[m] + 1), cid(I[m], J[m], K[m]), none(m), 4)
    quads = np.concatenate(quads).astype(np.int32)
    defs = [("inlet", "patch"), ("outlet", "patch"), ("walls", "wall"), ("sym1", "symmetry"), ("sym2", "symmetry")]
    return _assemble(points, quads, np.concatenate(ca).astype(np.int64), np.concatenate(cb).astype(np.int64),
                     np.concatenate(pf), defs, cc)


def annular_passage(nr=4, nt=4, nz=6, r0=0.2, r1=0.35, lz=0.3, n_sectors=5, sectors=1, stagger=0.35, lean=0.15, bulge=0.08):
    """Annular duct about the z axis, flow in +z: the shape of a turbomachinery passage (BASELINE config 5: DATurboFoam rotor,
    `cyclic` sides, MRF).  One passage spans 2*pi/n_sectors; `sectors` consecutive passages are generated.

    sectors < n_sectors: the two theta-sides are the patches `per_lo` / `per_hi`, type cyclic, transform rotational about z, face i of
    one coupled to face i of the other (the OpenFOAM convention).  sectors == n_sectors: the closed ring, no cyclic patches -- the
    periodic problem written out, which the parity tests use as the known answer for the cyclic mesh.
    The grid lines are staggered in theta along z (`stagger`, blade-passage like), lean with the radius (`lean`) and bulge inside a
    passage (`bulge`), the same way in every passage, so the mesh is non-orthogonal and skewed but exactly periodic.
    Cells are numbered passage-major: cell = s * (nr*nt*nz) + (ir + nr * (it + nt * iz))."""
    closed = sectors == n_sectors
    if sectors > n_sectors:
        raise ValueError("sectors > n_sectors")
    dth = 2.0 * np.pi / n_sectors
    NT = nt * sectors
    ntp = NT if closed else NT + 1  # point columns in theta

    def pid(i, j, k):
        return i + (nr + 1) * ((j % ntp if closed else j) + ntp * k)

    def cid(i, j, k):
        s_, jl = j // nt, j % nt
        return s_ * (nr * nt * nz) + i + nr * (jl + nt * k)

    rr = np.linspace(0.0, 1.0, nr + 1)
    zz = np.linspace(0.0, 1.0, nz + 1)
    points = np.empty(((nr + 1) * ntp * (nz + 1), 3))
    Ip, Jp, Kp = np.meshgrid(np.arange(nr + 1), np.arange(ntp), np.arange(nz + 1), indexing="ij")
    Ip, Jp, Kp = Ip.ravel(), Jp.ravel(), Kp.ravel()
    frac = (Jp % nt) / nt  # position inside the passage
    th = (Jp // nt) * dth + frac * dth + stagger * dth * np.sin(0.5 * np.pi * zz[Kp]) + lean * dth * rr[Ip] \
        + bulge * dth * np.sin(2.0 * np.pi * frac) * np.sin(np.pi * zz[Kp])
    rad = r0 + (r1 - r0) * (rr[Ip] + 0.06 * np.sin(np.pi * rr[Ip]) * np.cos(2.0 * np.pi * frac))
    zc = lz * (zz[Kp] + 0.05 * np.sin(np.pi * zz[Kp]) * np.sin(2.0 * np.pi * frac) * rr[Ip])
    idx = pid(Ip, Jp, Kp)
    points[idx, 0] = rad * np.cos(th)
    points[idx, 1] = rad * np.sin(th)
    points[idx, 2] = zc

    I, J, K = np.meshgrid(np.arange(nr), np.arange(NT), np.arange(nz), indexing="ij")
    I, J, K = I.ravel(), J.ravel(), K.ravel()
    corners = [pid(I + a, J + b, K + c) for a in (0, 1) for b in (0, 1) for c in (0, 1)]
    cc = np.zeros((nr * NT * nz, 3))
    cc[cid(I, J, K)] = sum(points[c] for c in corners) / 8.0

    quads, ca, cb, pf = [], [], [], []

    def add(q, a, b, patch):
        quads.append(np.stack(q, axis=1))
        ca.append(a)
        cb.append(b)
        pf.append(np.full(a.shape, patch, dtype=np.int64))

    def rface(i, j, k):
        return [pid(i, j, k), pid(i, j + 1, k), pid(i, j + 1, k + 1), pid(i, j, k + 1)]

    def tface(i, j, k):
        return [pid(i, j, k), pid(i + 1, j, k), pid(i + 1, j, k + 1), pid(i, j, k + 1)]

    def zface(i, j, k):
        return [pid(i, j, k), pid(i + 1, j, k), pid(i + 1, j + 1, k), pid(i, j + 1, k)]

    none = lambda m: np.full(int(m.sum()), -1)
    m = I >= 1
    add(rface(I[m], J[m], K[m]), cid(I[m] - 1, J[m], K[m]), cid(I[m], J[m], K[m]), -1)
    m = (J >= 1) | closed
    add(tface(I[m], J[m], K[m]), cid(I[m], (J[m] - 1) % NT, K[m]), cid(I[m], J[m], K[m]), -1)
    m = K >= 1
    add(zface(I[m], J[m], K[m]), cid(I[m], J[m], K[m] - 1), cid(I[m], J[m], K[m]), -1)
    m = K == 0
    add(zface(I[m], J[m], K[m]), cid(I[m], J[m], K[m]), none(m), 0)
    m = K == nz - 1
    add(zface(I[m], J[m], K[m] + 1), cid(I[m], J[m], K[m]), none(m), 1)
    m = I == 0
    add(rface(I[m], J[m], K[m]), cid(I[m], J[m], K[m]), none(m), 2)
    m = I == nr - 1
    add(rface(I[m] + 1, J[m], K[m]), cid(I[m], J[m], K[m]), none(m), 3)
    defs = [("inlet", "patch"), ("outlet", "patch"), ("hub", "wall"), ("shroud", "wall")]
    if not closed:
        m = J == 0
        add(tface(I[m], J[m], K[m]), cid(I[m], J[m], K[m]), none(m), 4)
        m = J == NT - 1
        add(tface(I[m], J[m] + 1, K[m]), cid(I[m], J[m], K[m]), none(m), 5)
        defs += [("per_lo", "cyclic"), ("per_hi", "cyclic")]
    quads = np.concatenate(quads).astype(np.int32)
    mesh = _assemble(points, quads, np.concatenate(ca).astype(np.int64), np.concatenate(cb).astype(np.int64), np.concatenate(pf), defs, cc)
    for pd in mesh.patches:
        if pd["type"] == "cyclic":
            pd.update(neighbourPatch="per_hi" if pd["name"] == "per_lo" else "per_lo", transform="rotational",
                      rotationAxis=(0.0, 0.0, 1.0), rotationCentre=(0.0, 0.0, 0.0))
    mesh.sector_angle = dth
    mesh.cells_per_sector = nr * nt * nz
    return mesh


def prism_channel(nx=10, ny=6, lx=2.0, ly=0.5, lz=0.1, contraction=0.3, skew=0.15):
    """The convergent channel meshed with triangular prisms (every quad column split along its diagonal): cells with
    5 faces, triangular and quadrilateral faces -- exercises the general polyhedral paths of the engine."""
    xs = np.linspace(0.0, lx, nx + 1)
    et = np.linspace(0.0, 1.0, ny + 1)
    h = ly * (1.0 - contraction * 0.5 * (1.0 - np.cos(np.pi * xs / lx)))
    Xg = xs[:, None] + skew * ly * np.sin(np.pi * et)[None, :] * np.sin(np.pi * xs / lx)[:, None]
    Yg = et[None, :] * h[:, None]

    def pid(i, j, k):
        return i + (nx + 1) * (j + (ny + 1) * k)

    points = np.empty(((nx + 1) * (ny + 1) * 2, 3))
    for k, z in enumerate((0.0, lz)):
        for j in range(ny + 1):
            for i in range(nx + 1):
                points[pid(i, j, k)] = (Xg[i, j], Yg[i, j], z)
    A = lambda i, j: 2 * (i + nx * j)       # prism on (p00, p10, p11)
    B = lambda i, j: 2 * (i + nx * j) + 1   # prism on (p00, p11, p01)
    faces, ca, cb, pf = [], [], [], []

    def add(pts, a, b, patch):
        faces.append(list(pts) + [-1] * (4 - len(pts)))
        ca.append(a)
        cb.append(b)
        pf.append(patch)

    for j in range(ny):
        for i in range(nx):
            p00, p10, p11, p01 = (i, j), (i + 1, j), (i + 1, j + 1), (i, j + 1)
            q = lambda p, k: pid(p[0], p[1], k)
            add([q(p00, 0), q(p11, 0), q(p11, 1), q(p00, 1)], A(i, j), B(i, j), -1)          # diagonal
            for k, patch in ((0, 3), (1, 4)):                                                   # z planes (triangles)
                add([q(p00, k), q(p10, k), q(p11, k)], A(i, j), -1, patch)
                add([q(p00, k), q(p11, k), q(p01, k)], B(i, j), -1, patch)
            # right edge of A: to B(i+1, j) or outlet
            add([q(p10, 0), q(p11, 0), q(p11, 1), q(p10, 1)], A(i, j), B(i + 1, j) if i + 1 < nx else -1, -1 if i + 1 < nx else 1)
            if i == 0:
                add([q(p00, 0), q(p01, 0), q(p01, 1), q(p00, 1)], B(i, j), -1, 0)                 # inlet
            # top edge of B: to A(i, j+1) or wall
            add([q(p01, 0), q(p11, 0), q(p11, 1), q(p01, 1)], B(i, j), A(i, j + 1) if j + 1 < ny else -1, -1 if j + 1 < ny else 2)
            if j == 0:
                add([q(p00, 0), q(p10, 0), q(p10, 1), q(p00, 1)], A(i, j), -1, 2)                 # lower wall
    faces = np.array(faces, dtype=np.int32)
    ca, cb, pf = np.array(ca, dtype=np.int64), np.array(cb, dtype=np.int64), np.array(pf, dtype=np.int64)
    # cell centres: mean of the 6 prism corners
    cc = np.zeros((2 * nx * ny, 3))
    for j in range(ny):
        for i in range(nx):
            c = [points[pid(a, b, k)] for (a, b) in ((i, j), (i + 1, j), (i + 1, j + 1)) for k in (0, 1)]
            cc[A(i, j)] = np.mean(c, axis=0)
            c = [points[pid(a, b, k)] for (a, b) in ((i, j), (i + 1, j + 1), (i, j + 1)) for k in (0, 1)]
            cc[B(i, j)] = np.mean(c, axis=0)
    defs = [("inlet", "patch"), ("outlet", "patch"), ("walls", "wall"), ("sym1", "symmetry"), ("sym2", "symmetry")]
    return _assemble(points, faces, ca, cb, pf, defs, cc)


# ----------------------------------------------------------------------------------------------
# OpenFOAM writers
# ----------------------------------------------------------------------------------------------

_HDR = """FoamFile
{{
    version     2.0;
    format      {fmt};
    class       {cls};
    location    "{loc}";
    object      {obj};
}}
"""


def _header(cls, loc, obj, fmt="ascii", note=None):
    s = _HDR.format(fmt=fmt, cls=cls, loc=loc, obj=obj)
    if note:
        s = s.replace("    object ", "    note        \"%s\";\n    object " % note)
    return s


def write_polymesh(case_dir, mesh: PolyMesh, binary=False):
    pm = os.path.join(case_dir, "constant", "polyMesh")
    os.makedirs(pm, exist_ok=True)
    fmt = "binary" if binary else "ascii"
    note = "nPoints:%d  nCells:%d  nFaces:%d  nInternalFaces:%d" % (
        mesh.n_points, mesh.n_cells, mesh.n_faces, mesh.n_internal_faces)
    # points
    with open(os.path.join(pm, "points"), "wb") as f:
        f.write(_header("vectorField", "constant/polyMesh", "points", fmt).encode())
        f.write(b"\n%d\n(" % mesh.n_points)
        if binary:
            f.write(mesh.points.tobytes())
        else:
            f.write(b"\n")
            f.write("\n".join("(%.17g %.17g %.17g)" % tuple(p) for p in mesh.points).encode())
            f.write(b"\n")
        f.write(b")\n")
    # faces
    with open(os.path.join(pm, "faces"), "wb") as f:
        if binary:
            # faceCompactList: offsets then flat labels
            f.write(_header("faceCompactList", "constant/polyMesh", "faces", fmt).encode())
            offs, labs = mesh.face_offsets_labels()
            f.write(b"\n%d\n(" % offs.size)
            f.write(offs.tobytes())
            f.write(b")\n\n%d\n(" % labs.size)
            f.write(labs.tobytes())
            f.write(b")\n")
        else:
            f.write(_header("faceList", "constant/polyMesh", "faces", fmt).encode())
            f.write(b"\n%d\n(\n" % mesh.n_faces)
            f.write("\n".join("%d(%s)" % ((q >= 0).sum(), " ".join(str(int(v)) for v in q if v >= 0)) for q in mesh.faces).encode())
            f.write(b"\n)\n")
    for name, arr in (("owner", mesh.owner), ("neighbour", mesh.neighbour)):
        with open(os.path.join(pm, name), "wb") as f:
            f.write(_header("labelList", "constant/polyMesh", name, fmt, note).encode())
            f.write(b"\n%d\n(" % arr.size)
            if binary:
                f.write(arr.astype(np.int32).tobytes())
            else:
                f.write(b"\n")
                f.write("\n".join(str(int(v)) for v in arr).encode())
                f.write(b"\n")
            f.write(b")\n")
    with open(os.path.join(pm, "boundary"), "w") as f:
        f.write(_header("polyBoundaryMesh", "constant/polyMesh", "boundary"))
        f.write("\n%d\n(\n" % len(mesh.patches))
        for p in mesh.patches:
            f.write("    %s\n    {\n        type            %s;\n" % (p["name"], p["type"]))
            if p["type"] == "wall":
                f.write("        inGroups        1(wall);\n")
            if p["type"] == "cyclic":
                f.write("        inGroups        1(cyclic);\n        neighbourPatch  %s;\n" % p["neighbourPatch"])
                if p.get("transform"):
                    f.write("        transform       %s;\n" % p["transform"])
                if "rotationAxis" in p:
                    f.write("        rotationAxis    (%.17g %.17g %.17g);\n" % tuple(p["rotationAxis"]))
                    f.write("        rotationCentre  (%.17g %.17g %.17g);\n" % tuple(p.get("rotationCentre", (0.0, 0.0, 0.0))))
                if "separationVector" in p:
                    f.write("        separationVector (%.17g %.17g %.17g);\n" % tuple(p["separationVector"]))
            f.write("        nFaces          %d;\n        startFace       %d;\n    }\n" % (p["size"], p["start"]))
        f.write(")\n")


def _fmt_val(v):
    if np.ndim(v) == 0:
        return "%.17g" % float(v)
    return "(" + " ".join("%.17g" % float(x) for x in v) + ")"


def write_field(case_dir, name, cls, dims, internal, bcs, time="0"):
    """internal: scalar/3-vector (uniform) or ndarray (nonuniform).  bcs: {patch: dict(type=..., ...)}."""
    d = os.path.join(case_dir, time)
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, name), "w") as f:
        f.write(_header(cls, time, name))
        f.write("\ndimensions      %s;\n\n" % dims)
        arr = np.asarray(internal, dtype=np.float64)
        is_vec = cls == "volVectorField"
        if (is_vec and arr.ndim == 1) or (not is_vec and arr.ndim == 0):
            f.write("internalField   uniform %s;\n\n" % _fmt_val(arr))
        else:
            f.write("internalField   nonuniform List<%s>\n%d\n(\n" % ("vector" if is_vec else "scalar", arr.shape[0]))
            if is_vec:
                f.write("\n".join("(%.17g %.17g %.17g)" % tuple(v) for v in arr))
            else:
                f.write("\n".join("%.17g" % v for v in arr))
            f.write("\n)\n;\n\n")
        f.write("boundaryField\n{\n")
        for patch, bc in bcs.items():
            f.write("    %s\n    {\n        type            %s;\n" % (patch, bc["type"]))
            for k, v in bc.items():
                if k == "type":
                    continue
                f.write("        %-15s uniform %s;\n" % (k, _fmt_val(np.asarray(v, dtype=np.float64))))
            f.write("    }\n")
        f.write("}\n")


def write_dicts(case_dir, nu=1.5e-5, ras_model="SpalartAllmaras", div_u="bounded Gauss linearUpwind grad(U)",
                div_nut="bounded Gauss upwind", relax_u=0.7, relax_p=0.3, relax_nut=0.7, consistent=False, transonic=False,
                div_phid_p="Gauss upwind", relax_p_eqn=None, relax_he=None):
    """relax_p_eqn: relaxationFactors.equations.p (pEqn.relax() of the transonic corrector); relax_he: equations e and h."""
    os.makedirs(os.path.join(case_dir, "constant"), exist_ok=True)
    os.makedirs(os.path.join(case_dir, "system"), exist_ok=True)
    with open(os.path.join(case_dir, "constant", "transportProperties"), "w") as f:
        f.write(_header("dictionary", "constant", "transportProperties"))
        f.write("\ntransportModel  Newtonian;\n\nnu              %.17g;\nPr 0.7;\nPrt 0.85;\n" % nu)
    with open(os.path.join(case_dir, "constant", "turbulenceProperties"), "w") as f:
        f.write(_header("dictionary", "constant", "turbulenceProperties"))
        f.write("\nsimulationType RAS;\nRAS\n{\n    RASModel        %s;\n    turbulence      on;\n    printCoeffs     off;\n}\n" % ras_model)
    with open(os.path.join(case_dir, "system", "fvSchemes"), "w") as f:
        f.write(_header("dictionary", "system", "fvSchemes"))
        f.write("""
ddtSchemes { default steadyState; }
gradSchemes { default Gauss linear; }
divSchemes
{
    default         none;
    div(phi,U)      %s;
    div(phi,nuTilda) %s;
    div((nuEff*dev2(T(grad(U))))) Gauss linear;
    div(phid,p)     %s;
    div(pc)         bounded Gauss upwind;
}
laplacianSchemes { default Gauss linear corrected; }
interpolationSchemes { default linear; }
snGradSchemes { default corrected; }
wallDist { method meshWaveFrozen; }
""" % (div_u, div_nut, div_phid_p))
    with open(os.path.join(case_dir, "system", "fvSolution"), "w") as f:
        f.write(_header("dictionary", "system", "fvSolution"))
        f.write("""
SIMPLE
{
    nNonOrthogonalCorrectors 0;
    consistent %s;
    transonic %s;
}
relaxationFactors
{
    fields { p %.17g; }
    equations { U %.17g; nuTilda %.17g;%s }
}
""" % ("true" if consistent else "false", "yes" if transonic else "no", relax_p, relax_u, relax_nut,
       ("" if relax_p_eqn is None else " p %.17g;" % relax_p_eqn) + ("" if relax_he is None else " e %.17g; h %.17g;" % (relax_he, relax_he))))
    with open(os.path.join(case_dir, "system", "controlDict"), "w") as f:
        f.write(_header("dictionary", "system", "controlDict"))
        f.write("\napplication simpleFoam;\nstartTime 0;\nendTime 1000;\ndeltaT 1;\n")


def default_bcs_naca(U0=(10.0, 0.0, 0.0), nuTilda0=4.5e-5, turbulent=True, wall_function=False):
    """Boundary conditions of the reference's NACA0012 incompressible case family
    (wing wall, inout farfield, symmetry planes)."""
    U0 = tuple(float(x) for x in U0)
    bcs = {
        "U": ("volVectorField", "[0 1 -1 0 0 0 0]", U0, {
            "wing": dict(type="fixedValue", value=(0.0, 0.0, 0.0)),
            "inout": dict(type="inletOutlet", inletValue=U0, value=U0),
            "sym1": dict(type="symmetry"), "sym2": dict(type="symmetry")}),
        "p": ("volScalarField", "[0 2 -2 0 0 0 0]", 0.0, {
            "wing": dict(type="zeroGradient"),
            "inout": dict(type="outletInlet", outletValue=0.0, value=0.0),
            "sym1": dict(type="symmetry"), "sym2": dict(type="symmetry")}),
    }
    if turbulent:
        bcs["nuTilda"] = ("volScalarField", "[0 2 -1 0 0 0 0]", nuTilda0, {
            "wing": dict(type="fixedValue", value=0.0),
            "inout": dict(type="inletOutlet", inletValue=nuTilda0, value=nuTilda0),
            "sym1": dict(type="symmetry"), "sym2": dict(type="symmetry")})
        bcs["nut"] = ("volScalarField", "[0 2 -1 0 0 0 0]", nuTilda0, {
            "wing": dict(type="nutUSpaldingWallFunction" if wall_function else "nutLowReWallFunction", value=0.0),
            "inout": dict(type="calculated", value=0.0),
            "sym1": dict(type="symmetry"), "sym2": dict(type="symmetry")})
    return bcs


def default_bcs_channel(U0=(10.0, 0.0, 0.0), nuTilda0=4.5e-5, turbulent=True):
    U0 = tuple(float(x) for x in U0)
    sym = {"sym1": dict(type="symmetry"), "sym2": dict(type="symmetry")}
    bcs = {
        "U": ("volVectorField", "[0 1 -1 0 0 0 0]", U0, dict(
            inlet=dict(type="fixedValue", value=U0), outlet=dict(type="inletOutlet", inletValue=(0.0, 0.0, 0.0), value=U0),
            walls=dict(type="fixedValue", value=(0.0, 0.0, 0.0)), **sym)),
        "p": ("volScalarField", "[0 2 -2 0 0 0 0]", 0.0, dict(
            inlet=dict(type="zeroGradient"), outlet=dict(type="fixedValue", value=0.0),
            walls=dict(type="zeroGradient"), **sym)),
    }
    if turbulent:
        bcs["nuTilda"] = ("volScalarField", "[0 2 -1 0 0 0 0]", nuTilda0, dict(
            inlet=dict(type="fixedValue", value=nuTilda0), outlet=dict(type="zeroGradient"),
            walls=dict(type="fixedValue", value=0.0), **sym))
        bcs["nut"] = ("volScalarField", "[0 2 -1 0 0 0 0]", nuTilda0, dict(
            inlet=dict(type="calculated", value=0.0), outlet=dict(type="calculated", value=0.0),
            walls=dict(type="nutLowReWallFunction", value=0.0), **sym))
    return bcs


def default_bcs_passage(Uin=(0.0, 0.0, 10.0), nuTilda0=4.5e-5, turbulent=True, cyclic=True):
    """Annular passage (annular_passage): axial inflow, fixed-pressure outflow, hub and shroud walls, cyclic sides."""
    Uin = tuple(float(x) for x in Uin)
    cyc = {"per_lo": dict(type="cyclic"), "per_hi": dict(type="cyclic")} if cyclic else {}
    wall0 = dict(type="fixedValue", value=(0.0, 0.0, 0.0))
    bcs = {
        "U": ("volVectorField", "[0 1 -1 0 0 0 0]", Uin, dict(
            inlet=dict(type="fixedValue", value=Uin), outlet=dict(type="inletOutlet", inletValue=(0.0, 0.0, 0.0), value=Uin),
            hub=dict(wall0), shroud=dict(wall0), **cyc)),
        "p": ("volScalarField", "[0 2 -2 0 0 0 0]", 0.0, dict(
            inlet=dict(type="zeroGradient"), outlet=dict(type="fixedValue", value=0.0),
            hub=dict(type="zeroGradient"), shroud=dict(type="zeroGradient"), **cyc)),
    }
    if turbulent:
        bcs["nuTilda"] = ("volScalarField", "[0 2 -1 0 0 0 0]", nuTilda0, dict(
            inlet=dict(type="fixedValue", value=nuTilda0), outlet=dict(type="zeroGradient"),
            hub=dict(type="fixedValue", value=0.0), shroud=dict(type="fixedValue", value=0.0), **cyc))
        bcs["nut"] = ("volScalarField", "[0 2 -1 0 0 0 0]", nuTilda0, dict(
            inlet=dict(type="calculated", value=0.0), outlet=dict(type="calculated", value=0.0),
            hub=dict(type="nutLowReWallFunction", value=0.0), shroud=dict(type="nutLowReWallFunction", value=0.0), **cyc))
    return bcs


def default_thermo(energy="sensibleInternalEnergy", transport="const", mu=1.8e-5, Pr=0.7, Prt=1.0, Cp=1005.0, molWeight=28.96,
                   divE="upwind", divEkp="upwind"):
    """thermophysicalProperties of the reference's DARhoSimpleFoam cases: hePsiThermo, pureMixture, perfectGas, hConst,
    const or sutherland transport (the combination DAResidual::updateThermoVars assumes, reference DAResidual.C:179-293)."""
    return dict(energy=energy, transport=transport, mu=mu, Pr=Pr, Prt=Prt, Cp=Cp, molWeight=molWeight, As=1.4792e-6, Ts=116.0,
                divE=divE, divEkp=divEkp)


def compressible_bcs(bcs, U0mag=None, p0=101325.0, T0=300.0):
    """Turn a default_bcs_* set into its compressible counterpart: absolute pressure level, a T field with the p-like
    role swapped (fixed where U is fixed/inflow, zero-gradient at walls/outflow)."""
    out = {k: (v[0], v[1], v[2], {pn: dict(pb) for pn, pb in v[3].items()}) for k, v in bcs.items()}
    cls, dims, _, pbs = out["p"]
    for pb in pbs.values():
        for key in ("value", "outletValue", "inletValue"):
            if key in pb:
                pb[key] = p0
    out["p"] = (cls, "[1 -1 -2 0 0 0 0]", p0, pbs)
    tb = {}
    for pn, ub in bcs["U"][3].items():
        ty = ub["type"]
        if ty == "symmetry":
            tb[pn] = dict(type="symmetry")
        elif ty == "cyclic":
            tb[pn] = dict(type="cyclic")
        elif ty == "inletOutlet":
            tb[pn] = dict(type="inletOutlet", inletValue=T0, value=T0)
        elif ty == "fixedValue" and any(abs(x) > 0 for x in ub["value"]):
            tb[pn] = dict(type="fixedValue", value=T0)
        else:
            tb[pn] = dict(type="zeroGradient")
    out["T"] = ("volScalarField", "[0 0 0 1 0 0 0]", T0, tb)
    return out


def write_thermo(case_dir, thermo):
    with open(os.path.join(case_dir, "constant", "thermophysicalProperties"), "w") as f:
        f.write(_header("dictionary", "constant", "thermophysicalProperties"))
        tr = "sutherland" if thermo["transport"] == "sutherland" else "const"
        f.write("""
thermoType
{
    type            hePsiThermo;
    mixture         pureMixture;
    transport       %s;
    thermo          hConst;
    equationOfState perfectGas;
    specie          specie;
    energy          %s;
}
mixture
{
    specie { molWeight %.17g; }
    thermodynamics { Cp %.17g; Hf 0; gamma %.17g; }
    transport { mu %.17g; Pr %.17g; As %.17g; Ts %.17g; }
}
Prt %.17g;
""" % (tr, thermo["energy"], thermo["molWeight"], thermo["Cp"], thermo.get("gamma", 1.4), thermo["mu"], thermo["Pr"], thermo["As"], thermo["Ts"], thermo["Prt"]))
    # compressible convection schemes next to the incompressible ones
    path = os.path.join(case_dir, "system", "fvSchemes")
    txt = open(path).read()
    sch = {"upwind": "bounded Gauss upwind", "linear": "bounded Gauss linear", "linearUpwind": "bounded Gauss linearUpwind grad(e)"}
    he = "e" if thermo["energy"] == "sensibleInternalEnergy" else "h"
    extra = "    div(phi,%s)      %s;\n    div(phi,%s)    %s;\n    div(((rho*nuEff)*dev2(T(grad(U))))) Gauss linear;\n" % (
        he, sch[thermo["divE"]], "Ekp" if he == "e" else "K", sch[thermo["divEkp"]])
    txt = txt.replace("    div(pc)         bounded Gauss upwind;\n", extra + "    div(pc)         bounded Gauss upwind;\n")
    open(path, "w").write(txt)


def write_case(case_dir, mesh: PolyMesh, bcs, binary=False, **dict_kw):
    """Write polyMesh + 0/ fields + dictionaries.  `bcs` as returned by default_bcs_*."""
    write_polymesh(case_dir, mesh, binary=binary)
    for name, (cls, dims, internal, patch_bcs) in bcs.items():
        write_field(case_dir, name, cls, dims, internal, patch_bcs)
    ras = "SpalartAllmaras" if "nuTilda" in bcs else "dummy"
    dict_kw.setdefault("ras_model", ras)
    thermo = dict_kw.pop("thermo", None)
    mrf = dict_kw.pop("mrf", None)
    write_dicts(case_dir, **dict_kw)
    if thermo is not None:
        write_thermo(case_dir, thermo)
    if mrf is not None:
        write_mrf(case_dir, mrf)
    return case_dir


def write_mrf(case_dir, mrf):
    """constant/MRFProperties + constant/polyMesh/cellZones of one rotating zone.  mrf = dict(cellZone=name, cells=[...],
    origin=(3), axis=(3), omega=rad/s, nonRotatingPatches=[...]) -- the entries of OpenFOAM's MRFZone dictionary."""
    cells = np.asarray(mrf["cells"], dtype=np.int64)
    with open(os.path.join(case_dir, "constant", "polyMesh", "cellZones"), "w") as f:
        f.write(_header("regIOobject", "constant/polyMesh", "cellZones"))
        f.write("\n1\n(\n%s\n{\n    type cellZone;\n    cellLabels List<label> %d\n(\n%s\n);\n}\n)\n" % (
            mrf["cellZone"], cells.size, "\n".join(str(int(c)) for c in cells)))
    with open(os.path.join(case_dir, "constant", "MRFProperties"), "w") as f:
        f.write(_header("dictionary", "constant", "MRFProperties"))
        f.write("\nMRF\n{\n    cellZone %s;\n    active yes;\n    nonRotatingPatches (%s);\n    origin (%.17g %.17g %.17g);\n"
                "    axis (%.17g %.17g %.17g);\n    omega %.17g;\n}\n" % ((mrf["cellZone"], " ".join(mrf.get("nonRotatingPatches", [])))
                                                                         + tuple(mrf["origin"]) + tuple(mrf["axis"]) + (mrf["omega"],)))


# ----------------------------------------------------------------------------------------------
# synthetic states
# ----------------------------------------------------------------------------------------------


def quad_face_geometry(mesh: PolyMesh):
    """Area vectors and centres of quad faces (diagonal cross product / vertex mean): good enough to
    synthesise a face-flux field; the engine computes the exact OpenFOAM geometry itself."""
    fa = mesh.faces.copy()
    tri = fa[:, 3] < 0
    fa[tri, 3] = fa[tri, 0]
    p = mesh.points[fa]
    Sf = 0.5 * np.cross(p[:, 2] - p[:, 0], p[:, 3] - p[:, 1])
    return Sf, p.mean(axis=1)


def to_compressible_state(mesh: PolyMesh, W, thermo, p0=101325.0, T0=300.0, turbulent=True):
    """[U|p|nuTilda|phi] -> [U|p0+p|T|nuTilda|rho_f*phi] (DARhoSimpleFoam ordering, mass flux) with a smooth temperature field."""
    nC, nF, nIF = mesh.n_cells, mesh.n_faces, mesh.n_internal_faces
    Rg = 8314.4700665 / thermo["molWeight"]
    U = W[:3 * nC]
    p = p0 + W[3 * nC:4 * nC]
    off = 4 * nC
    nt = None
    if turbulent:
        nt = W[off:off + nC]
        off += nC
    phi = W[off:off + nF]
    Um2 = (U.reshape(nC, 3) ** 2).sum(axis=1)
    Tt = T0 - 0.5 * Um2 / thermo["Cp"] * 0.8  # roughly constant total temperature
    rho = p / (Rg * Tt)
    rf = np.empty(nF)
    rf[:nIF] = 0.5 * (rho[mesh.owner[:nIF]] + rho[mesh.neighbour])
    rf[nIF:] = rho[mesh.owner[nIF:]]
    parts = [U, p, Tt]
    if turbulent:
        parts.append(nt)
    parts.append(phi * rf)
    return np.concatenate(parts)


def boundary_layer_state(mesh: PolyMesh, yWall, U0=(10.0, 0.0, 0.0), nuTilda0=4.5e-5, delta=0.02, turbulent=True,
                         seed=1234, noise=0.0):
    """Smooth analytic state in the reference's state ordering (SURVEY.md section 8d): a velocity
    profile U0*(1-exp(-y/delta)) in the wall distance y, a pressure bump, a nuTilda hump inside the
    layer, phi = U_f . S_f with zero flux through walls and symmetry planes; optional seeded noise."""
    nC, nF, nIF = mesh.n_cells, mesh.n_faces, mesh.n_internal_faces
    rng = np.random.default_rng(seed)
    Sf, Cf = quad_face_geometry(mesh)
    # cell centres as the mean of the cell's face centres
    C = np.zeros((nC, 3))
    cnt = np.zeros(nC)
    np.add.at(C, mesh.owner, Cf)
    np.add.at(cnt, mesh.owner, 1.0)
    np.add.at(C, mesh.neighbour, Cf[:nIF])
    np.add.at(cnt, mesh.neighbour, 1.0)
    C /= cnt[:, None]
    U0 = np.asarray(U0, dtype=np.float64)
    prof = 1.0 - np.exp(-np.asarray(yWall) / delta)
    U = U0[None, :] * prof[:, None]
    p = 0.15 * float(U0 @ U0) * np.exp(-((C[:, 0] - 0.5) ** 2 + C[:, 1] ** 2) / 0.5)
    nt = nuTilda0 * (1.0 + 20.0 * np.exp(-yWall / delta) * (1.0 - np.exp(-yWall / (0.1 * delta))))
    if noise > 0.0:
        U *= 1.0 + noise * rng.uniform(-1, 1, U.shape)
        p *= 1.0 + noise * rng.uniform(-1, 1, nC)
        nt *= 1.0 + noise * rng.uniform(-1, 1, nC)
    Uf = np.empty((nF, 3))
    Uf[:nIF] = 0.5 * (U[mesh.owner[:nIF]] + U[mesh.neighbour])
    Uf[nIF:] = U[mesh.owner[nIF:]]
    phi = np.einsum("ij,ij->i", Uf, Sf)
    for pch in mesh.patches:
        if pch["type"] in ("symmetry", "wall"):
            phi[pch["start"]:pch["start"] + pch["size"]] = 0.0
    parts = [U.ravel(), p]
    if turbulent:
        parts.append(nt)
    parts.append(phi)
    return np.concatenate(parts)


def merged_face_order(mesh: PolyMesh):
    """Face numbering of the engine on a mesh with cyclic patches (csrc/mesh.hpp mergeCyclics): the internal faces, then ONE face per
    coupled pair (the face of the first patch of the pair: owner = its cell, neighbour = the cell on the partner patch), then the
    faces of the other patches.  Returns the polyMesh face index of every engine face; phi of a coupled face is the flux out of the
    first patch.  Meshes without cyclic patches: the identity."""
    names = [p["name"] for p in mesh.patches]
    parts = [np.arange(mesh.n_internal_faces)]
    for pi, p in enumerate(mesh.patches):
        if p["type"] == "cyclic" and names.index(p["neighbourPatch"]) > pi:
            parts.append(np.arange(p["start"], p["start"] + p["size"]))
    for p in mesh.patches:
        if p["type"] != "cyclic":
            parts.append(np.arange(p["start"], p["start"] + p["size"]))
    return np.concatenate(parts)


def passage_state(mesh: PolyMesh, Uax=10.0, nuTilda0=4.5e-5, thermo=None, p0=101325.0, T0=300.0, seed=1234, noise=0.001, r0=0.2, r1=0.35,
                  n_sectors=None):
    """Synthetic flow through annular_passage(): axial velocity with a hub-to-shroud profile, swirl, passage-periodic pressure
    and temperature fields (+ seeded noise), flux = rho_f U_f . Sf.  Returned in the ENGINE's ordering ([U | p | (T) | nuTilda | phi],
    phi over merged_face_order(mesh)); the state of a periodic image is the rotated state, so the field repeats by construction."""
    rng = np.random.default_rng(seed)
    Sf, Cf = quad_face_geometry(mesh)
    nC, nIF = mesh.n_cells, mesh.n_internal_faces
    cnt = np.bincount(mesh.owner, minlength=nC) + np.bincount(mesh.neighbour, minlength=nC)
    C = np.stack([np.bincount(mesh.owner, weights=Cf[:, k], minlength=nC) + np.bincount(mesh.neighbour, weights=Cf[:nIF, k], minlength=nC)
                  for k in range(3)], axis=1) / cnt[:, None]
    ns_ = n_sectors if n_sectors is not None else int(round(2.0 * np.pi / mesh.sector_angle))
    r, th, z = np.hypot(C[:, 0], C[:, 1]), np.arctan2(C[:, 1], C[:, 0]), C[:, 2]
    eta = np.clip((r - r0) / (r1 - r0), 0.0, 1.0)
    prof = 4.0 * eta * (1.0 - eta) + 0.05
    ur = 0.02 * Uax * np.sin(ns_ * th) * np.sin(np.pi * eta)
    ut = 0.3 * Uax * prof * (1.0 + 0.1 * np.cos(ns_ * th))
    uz = Uax * prof * (1.0 + 0.05 * np.sin(ns_ * th + 3.0 * z))
    U = np.stack([ur * np.cos(th) - ut * np.sin(th), ur * np.sin(th) + ut * np.cos(th), uz], axis=1)
    U *= 1.0 + noise * rng.uniform(-1, 1, U.shape)
    zl = z / max(z.max(), 1e-300)
    p = 0.5 * Uax**2 * ((1.0 - zl) + 0.1 * np.cos(ns_ * th) * eta) * (1.0 + noise * rng.uniform(-1, 1, nC))
    nt = nuTilda0 * (1.0 + 3.0 * prof) * (1.0 + noise * rng.uniform(-1, 1, nC))
    rho = np.ones(nC)
    parts = [U.ravel()]
    if thermo is not None:
        p = p0 + p
        T = T0 * (1.0 + 0.02 * np.sin(ns_ * th) * np.cos(9.0 * z)) * (1.0 + 0.1 * noise * rng.uniform(-1, 1, nC))
        rho = p / (8314.4700665 / thermo["molWeight"] * T)
        parts += [p, T]
    else:
        parts.append(p)
    parts.append(nt)
    nei = np.concatenate([mesh.neighbour, mesh.owner[nIF:]])
    phi = 0.5 * (rho[mesh.owner] + rho[nei]) * np.einsum("ij,ij->i", 0.5 * (U[mesh.owner] + U[nei]), Sf)
    phi *= 1.0 + noise * rng.uniform(-1, 1, phi.size)
    for pch in mesh.patches:
        if pch["type"] == "wall":
            phi[pch["start"]:pch["start"] + pch["size"]] = 0.0
    parts.append(phi[merged_face_order(mesh)])
    return np.concatenate(parts)
