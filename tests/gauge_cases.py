"""Cases shared by the CPU and GPU tiers of the gauge half of an HMC step: path tables generated from geometry, SU(3)
link fields, the numpy restatement of the force, the update, the momentum action and the plaquette, the reference's own
host gauge force (oracle/_ref/libquda_gaugeref.so, where it was built) and one runner for the host twin and the library.

Conventions (quda_b200/gauge.py): links QDP [4][V][3][3][2], parity-major sites; mom [V][4][10]; a path is a list of steps,
d in 0..3 forward along d and 7 - d backward along d, walked from x + mu-hat back to x; internally the restatement works on
the lexicographic complex fields of tests/clover_build_ref.py."""
import ctypes as C
import os

import numpy as np

import clover_build_ref as R
import clover_force_ref as CF
from quda_b200 import fields as F
from quda_b200 import lib as L

REF_SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libquda_gaugeref.so")


# ------------------------------------------------------------------ path tables
def _enc(step):
    """(+1 or -1) * (d + 1) -> the reference's step code"""
    d = abs(step) - 1
    return d if step > 0 else 7 - d


def _paths(loops):
    """loops[mu]: closed loops as signed steps, each starting with +mu at x -> paths[mu] (the steps after U_mu(x))"""
    return [[[_enc(s) for s in loop[1:]] for loop in loops[mu]] for mu in range(4)]


def plaquette_loops(mu):
    return [[mu + 1, s * (nu + 1), -(mu + 1), -s * (nu + 1)] for nu in range(4) if nu != mu for s in (1, -1)]


def rectangle_loops(mu):
    out = []
    for nu in range(4):
        if nu == mu:
            continue
        for s in (1, -1):
            m, n = mu + 1, s * (nu + 1)
            out += [[m, m, n, -m, -m, -n], [m, n, -m, -m, -n, m], [m, n, n, -m, -n, -n]]
    return out


def parallelogram_loops(mu):
    out = []
    for nu in range(4):
        for rho in range(4):
            if len({mu, nu, rho}) < 3:
                continue
            for sn in (1, -1):
                for sr in (1, -1):
                    m, n, r = mu + 1, sn * (nu + 1), sr * (rho + 1)
                    out.append([m, n, r, -m, -n, -r])
    return out


def path_set(name):
    """(paths[mu][i], coefficients) of 'plaq' (6 per direction), 'plaq+rect' (6 + 18) or 'symanzik48' (+ 24 parallelograms)"""
    kinds = {"plaq": [plaquette_loops], "plaq+rect": [plaquette_loops, rectangle_loops],
             "symanzik48": [plaquette_loops, rectangle_loops, parallelogram_loops]}[name]
    coeff = {plaquette_loops: 1.0, rectangle_loops: -1.0 / 12, parallelogram_loops: 0.03}
    loops = [sum((k(mu) for k in kinds), []) for mu in range(4)]
    coeffs = sum(([coeff[k]] * len(k(0)) for k in kinds), [])
    return _paths(loops), coeffs


# ------------------------------------------------------------------ fields
def _su3_from_unitary(q):
    return q / np.linalg.det(q)[..., None, None] ** (1.0 / 3)


def haar_links(X, seed):
    rng = np.random.default_rng(seed)
    V = int(np.prod(X))
    z = (rng.normal(size=(4, V, 3, 3)) + 1j * rng.normal(size=(4, V, 3, 3))) / np.sqrt(2)
    q, r = np.linalg.qr(z)
    d = np.diagonal(r, axis1=-2, axis2=-1)
    q = q * (d / np.abs(d))[..., None, :]
    return to_qdp(_su3_from_unitary(q))


def expm_ah(A):
    """exp of anti-Hermitian matrices [..][3][3] by eigendecomposition"""
    w, v = np.linalg.eigh(-1j * A)
    return np.einsum("...ij,...j,...kj->...ik", v, np.exp(1j * w), v.conj())


def near_identity_links(X, seed, eps=0.1):
    rng = np.random.default_rng(seed)
    V = int(np.prod(X))
    H = CF.ta(rng.normal(size=(4, V, 3, 3)) + 1j * rng.normal(size=(4, V, 3, 3)))
    return to_qdp(expm_ah(eps * H))


def to_qdp(U):
    return np.ascontiguousarray(np.stack([U.real, U.imag], -1))


def cplx(gauge):
    g = np.asarray(gauge, dtype=np.float64)
    return g[..., 0] + 1j * g[..., 1]


def antiperiodic(gauge, X):
    """the links with the fermion boundary sign: U_t(x) * -1 on the last time slice"""
    g = np.array(gauge)
    for p in range(2):
        c = F.cb_coords(X, p)
        Vh = len(c)
        idx = p * Vh + np.nonzero(c[:, 3] == X[3] - 1)[0]
        g[3, idx] *= -1
    return g


def random_mom(V, seed, scale=1.0):
    """traceless anti-Hermitian momenta [V][4][10], Gaussian in the mom_action normalisation times scale"""
    rng = np.random.default_rng(seed)
    return scale * CF.mom_from_matrices(CF.ta(rng.normal(size=(V, 4, 3, 3)) + 1j * rng.normal(size=(V, 4, 3, 3))))


# ------------------------------------------------------------------ numpy restatement
def _at(a, off):
    for d in range(4):
        if off[d]:
            a = R.shift(a, d, off[d])
    return a


def path_field(U, mu, path):
    """lex [t][z][y][x][3][3]: the ordered product of the links of path walked from x + mu-hat"""
    off = [0, 0, 0, 0]
    off[mu] = 1
    M = None
    for st in path:
        if st < 4:
            L_ = _at(U[st], off)
            off[st] += 1
        else:
            d = 7 - st
            off[d] -= 1
            L_ = R.dag(_at(U[d], off))
        M = L_ if M is None else M @ L_
    return M


def staple_sum(gauge, X, paths, coeffs, mu):
    U = R.links(gauge, X)
    return U[mu] @ sum(c * path_field(U, mu, p) for c, p in zip(coeffs, paths[mu]))


def force(mom, gauge, X, paths, coeffs, eb3):
    """mom <- TA(mom - eb3 U_mu(x) sum_i c_i path_i)"""
    m = CF.mom_to_matrices(mom)
    for mu in range(4):
        W = R.from_lex(staple_sum(gauge, X, paths, coeffs, mu), X)
        m[:, mu] = CF.ta(m[:, mu] - eb3 * W)
    return CF.mom_from_matrices(m)


def loop_action(gauge, X, paths, coeffs, beta):
    """beta sum over loops c (1 - Re tr / 3), every loop once: loop i passes len(path_i) + 1 links, each of which sees it"""
    U = R.links(gauge, X)
    S = 0.0
    for mu in range(4):
        for c, p in zip(coeffs, paths[mu]):
            tr = np.trace(U[mu] @ path_field(U, mu, p), axis1=-2, axis2=-1).real
            S += beta * c * np.sum(1.0 - tr / 3.0) / (len(p) + 1)
    return S


def plaquette(gauge, X):
    """(total, spatial, temporal) means of Re tr U_P / 3"""
    U = R.links(gauge, X)
    s, t = [], []
    for mu in range(4):
        for nu in range(mu + 1, 4):
            P = U[mu] @ R.shift(U[nu], mu, 1) @ R.dag(R.shift(U[mu], nu, 1)) @ R.dag(U[nu])
            (t if nu == 3 else s).append(np.trace(P, axis1=-2, axis2=-1).real.mean() / 3)
    sp, tm = np.mean(s), np.mean(t)
    return 0.5 * (sp + tm), sp, tm


def mom_action(mom):
    m = np.asarray(mom, dtype=np.float64)
    return float(np.sum(m[..., :6] ** 2) + 0.5 * np.sum(m[..., 6:9] ** 2) - 4.0 * (m.size // 10))


def traceless_p(mom, conj_mom=False):
    """P [V][4][3][3]: the traceless part of mom (of its adjoint with conj_mom)"""
    m = CF.mom_to_matrices(mom)
    m = m - (np.trace(m, axis1=-2, axis2=-1) / 3)[..., None, None] * np.eye(3)
    return -m if conj_mom else m


def deviation(got, want, base):
    """largest |got - want| relative to the largest entry of the change want - base"""
    return np.abs(got - want).max() / np.abs(want - base).max()


# ------------------------------------------------------------------ the reference's host gauge force
def have_ref():
    return os.path.exists(REF_SO)


_ref = None


def ref_lib():
    global _ref
    if _ref is None:
        _ref = C.CDLL(REF_SO)
        _ref.ref_gauge_force.restype = None
        _ref.ref_mom_action.restype = C.c_double
    return _ref


def ref_force(mom, gauge, X, paths, coeffs, eb3):
    lib = ref_lib()
    Xc = (C.c_int * 4)(*X)
    lib.ref_set_dims(Xc)
    from quda_b200 import gauge as G
    table, lengths, n, max_length = G.path_table(paths)
    m = np.ascontiguousarray(mom, dtype=np.float64).copy()
    g = np.ascontiguousarray(gauge, dtype=np.float64)
    gp = (C.c_void_p * 4)(*[g[mu].ctypes.data for mu in range(4)])
    lib.ref_gauge_force(C.c_void_p(m.ctypes.data), gp, Xc, table.ctypes.data_as(C.c_void_p), (C.c_int * n)(*lengths),
                        (C.c_double * n)(*coeffs), C.c_int(n), C.c_int(max_length), C.c_double(eb3))
    return m


def ref_mom_action(mom):
    m = np.ascontiguousarray(mom)
    return ref_lib().ref_mom_action(C.c_void_p(m.ctypes.data), C.c_int(m.dtype.itemsize), C.c_int(m.size // 10))


# ------------------------------------------------------------------ one runner for the twin (numpy) and the library (torch)
class Runner:
    """Calls the four entry points of `lib` with prefix `prefix` on numpy inputs; dev=True puts the fields on the GPU"""

    def __init__(self, lib, prefix, dev=False):
        self.lib, self.prefix, self.dev = lib, prefix, dev

    def _put(self, a):
        a = np.ascontiguousarray(a).copy()
        if self.dev:
            import torch
            return torch.from_numpy(a).cuda()
        return a

    def _ptr(self, t):
        return t.data_ptr() if self.dev else t.ctypes.data

    def _get(self, t):
        return t.cpu().numpy() if self.dev else t

    def _links(self, g):
        return (C.c_void_p * 4)(*[self._ptr(g[mu]) for mu in range(4)])

    def _fn(self, name):
        return getattr(self.lib, self.prefix + "_" + name)

    def check(self, rc):
        L.check(rc, self.lib, self.prefix)

    def force_rc(self, mom, gauge, X, table, lengths, coeffs, n, max_length, eb3, prec):
        dt = np.float64 if prec == 8 else np.float32
        m, g = self._put(np.asarray(mom, dtype=dt)), self._put(np.asarray(gauge, dtype=dt))
        t = np.ascontiguousarray(table, dtype=np.int32)
        rc = self._fn("gauge_force")(self._ptr(m), self._links(g), (C.c_int * 4)(*X), prec, t.ctypes.data_as(C.POINTER(C.c_int)),
                                     (C.c_int * len(lengths))(*lengths), (C.c_double * len(coeffs))(*coeffs), n, max_length,
                                     float(eb3), None)
        return rc, self._get(m)

    def force(self, mom, gauge, X, paths, coeffs, eb3, prec=8):
        from quda_b200 import gauge as G
        table, lengths, n, max_length = G.path_table(paths)
        rc, m = self.force_rc(mom, gauge, X, table, lengths, coeffs, n, max_length, eb3, prec)
        self.check(rc)
        return m

    def update(self, gauge, mom, X, dt, conj_mom=False, exact=True, prec=8, in_place=False):
        typ = np.float64 if prec == 8 else np.float32
        g, m = self._put(np.asarray(gauge, dtype=typ)), self._put(np.asarray(mom, dtype=typ))
        out = g if in_place else self._put(np.zeros_like(np.asarray(gauge, dtype=typ)))
        self.check(self._fn("update_gauge")(self._links(out), self._links(g), self._ptr(m), (C.c_int * 4)(*X), prec, float(dt),
                                            int(conj_mom), int(exact), None))
        return self._get(out)

    def mom_action(self, mom, X, prec=8):
        m = self._put(np.asarray(mom, dtype=np.float64 if prec == 8 else np.float32))
        S = C.c_double()
        self.check(self._fn("mom_action")(C.byref(S), self._ptr(m), (C.c_int * 4)(*X), prec, None))
        return S.value

    def plaquette(self, gauge, X, prec=8):
        g = self._put(np.asarray(gauge, dtype=np.float64 if prec == 8 else np.float32))
        p = (C.c_double * 3)()
        self.check(self._fn("plaquette")(p, self._links(g), (C.c_int * 4)(*X), prec, None))
        return tuple(p)


SHAPES = [(4, 4, 4, 4), (4, 6, 8, 10), (2, 4, 4, 6), (4, 4, 6, 2), (6, 2, 4, 6)]  # the last: Vh = 144, not a multiple of 128
PATH_SETS = ["plaq", "plaq+rect", "symanzik48"]
FIELDS = {"near_identity": lambda X, s: near_identity_links(X, s, 0.1), "haar": haar_links}
