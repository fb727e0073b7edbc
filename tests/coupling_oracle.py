"""ctypes wrapper of tests/coupling_oracle.cpp: the face force vectors of forceCouplingOutput and their tapes, evaluated on an
oracle.pyoracle.Oracle's case.  TEST INFRASTRUCTURE ONLY.

The library is compiled on first use with the oracle's compiler flags into the temporary directory (keyed by a hash of its
sources, so a read-only tree and repeated sessions work)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SOURCES = [os.path.join(_HERE, "coupling_oracle.cpp"), os.path.join(_HERE, "..", "oracle", "oracle.cpp"),
            os.path.join(_HERE, "..", "oracle", "tape.hpp")]
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        h = hashlib.sha256()
        for s in _SOURCES:
            with open(s, "rb") as f:
                h.update(f.read())
        so = os.path.join(tempfile.gettempdir(), "dab_coupling_oracle_%s.so" % h.hexdigest()[:16])
        if not os.path.exists(so):
            tmp = "%s.%d.tmp" % (so, os.getpid())
            subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-fPIC", "-shared", "-o", tmp, _SOURCES[0]])
            os.replace(tmp, so)
        _LIB = C.CDLL(so)
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _mask(patches):
    m = 0
    for p in patches:
        m |= 1 << int(p)
    return m


def face_forces(orc, W, patches, pRef=0.0):
    """[nBF, 3] wall force vectors Sf (p_b - pRef) + Sf & devRhoReff_b of the faces of the listed patch indices (zero elsewhere)."""
    W = np.ascontiguousarray(W, dtype=np.float64)
    out = np.zeros(3 * (orc.mesh.n_faces - orc.mesh.n_internal_faces))
    lib().cpl_face_forces(orc.h, _p(W), C.c_uint(_mask(patches)), C.c_double(pRef), _p(out))
    return out.reshape(-1, 3)


def face_forces_jtvec(orc, W, patches, seeds, wrt="states", pRef=0.0, normalize=True):
    """Tape of sum_b seeds[b] . F_b (seeds [nBF, 3]) against the states (scaled like the reference) or, wrt="points", the mesh
    points through the geometry."""
    W = np.ascontiguousarray(W, dtype=np.float64)
    sd = np.ascontiguousarray(seeds, dtype=np.float64).ravel()
    out = np.zeros(orc.ndof if wrt == "states" else 3 * orc.mesh.n_points)
    lib().cpl_face_forces_jtvec(orc.h, _p(W), C.c_uint(_mask(patches)), C.c_double(pRef), _p(sd), C.c_int(0 if wrt == "states" else 1),
                                C.c_int(int(normalize)), _p(out))
    return out
