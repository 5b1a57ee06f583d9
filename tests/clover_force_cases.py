"""Cases shared by the CPU and GPU tiers of the clover force: random full-lattice spinor pairs, coefficients and momenta,
the per-piece coefficient sets, the call of b200_clover_force_accumulate on a backend (the host twin or the library) and
the comparison with the numpy restatement (tests/clover_force_ref.py)."""
import ctypes as C

import numpy as np

import clover_build_ref as R
import clover_force_ref as CF
import oracle
from quda_b200 import fields as F
from quda_b200 import lib as L

PIECES = ["hop", "sigma", "trace", "all"]


class Case:
    """n spinor pairs (DeGrand-Rossi host order, both parities), links, A, mom and coefficients on lattice X"""

    def __init__(self, X, n, seed=7, csw_kappa=0.12 * 1.3):
        self.X, self.n = tuple(X), n
        V = int(np.prod(X))
        self.gauge = oracle.random_gauge(X, 8, seed=seed, antiperiodic_t=True)
        self.packed = R.compute_clover(self.gauge, X, csw_kappa)
        self.xs = [oracle.random_spinor(X, 8, seed=seed + 10 + i, nparity=2) - 0.5 for i in range(n)]
        self.ps = [oracle.random_spinor(X, 8, seed=seed + 100 + i, nparity=2) - 0.5 for i in range(n)]
        rng = np.random.default_rng(seed)
        # the update is of the size of mom, so that the comparison measures the force rather than the storage of mom
        self.mom = 0.1 * CF.mom_from_matrices(CF.ta(rng.normal(size=(V, 4, 3, 3)) + 1j * rng.normal(size=(V, 4, 3, 3))))
        self.fc = list(rng.uniform(-1.0, 1.0, n))
        self.eps = [tuple(rng.uniform(-0.5, 0.5, 2)) for _ in range(n)]
        self.sigma_coeff = 0.5
        self.trlog_parity = 1

    def coefficients(self, piece):
        z = [0.0] * self.n
        fc = self.fc if piece in ("hop", "all") else z
        eps = self.eps if piece in ("sigma", "all") else [(0.0, 0.0)] * self.n
        sc = self.sigma_coeff if piece in ("trace", "all") else 0.0
        return fc, eps, sc

    def reference(self, piece):
        fc, eps, sc = self.coefficients(piece)
        xl = [CF.host_to_lex(x, self.X) for x in self.xs]
        pl = [CF.host_to_lex(p, self.X) for p in self.ps]
        return CF.accumulate(self.mom, self.gauge, self.packed, xl, pl, fc, eps, sc, self.trlog_parity, self.X)

    def native(self, host, prec):
        """full-lattice host spinor -> native bytes (both parity blocks)"""
        Vh = F.volume_cb(self.X)
        return np.concatenate([F.spinor_to_native(host[p * Vh:(p + 1) * Vh], prec) for p in range(2)])


def run(lib, prefix, case, piece, prec, to_dev=lambda a: a, to_host=lambda a: a, ptr=lambda a: a.ctypes.data):
    """mom after b200_clover_force_accumulate (prefix "b200" or "twin") on the fields of `case`, as float64 [V][4][10]"""
    dt = oracle._dt(prec)
    fc, eps, sc = case.coefficients(piece)
    mom = to_dev(case.mom.astype(dt))
    gauge = to_dev(np.ascontiguousarray(case.gauge.astype(dt)))
    packed = to_dev(np.ascontiguousarray(case.packed.astype(dt)))
    xs = [to_dev(case.native(x, prec)) for x in case.xs]
    ps = [to_dev(case.native(p, prec)) for p in case.ps]
    q = (C.c_void_p * 4)(*[ptr(gauge[mu]) for mu in range(4)])
    xa = (C.c_void_p * case.n)(*[ptr(x) for x in xs])
    pa = (C.c_void_p * case.n)(*[ptr(p) for p in ps])
    rc = getattr(lib, prefix + "_clover_force_accumulate")(
        ptr(mom), q, ptr(packed), (C.c_int * 4)(*case.X), prec, case.n, xa, pa, (C.c_double * case.n)(*fc),
        (C.c_double * (2 * case.n))(*[v for e in eps for v in e]), sc, case.trlog_parity, None)
    L.check(rc, lib, prefix)
    return np.asarray(to_host(mom), dtype=np.float64)


def deviation(got, want, mom0):
    """largest |got - want| relative to the largest entry of the update"""
    return np.abs(got - want).max() / np.abs(want - mom0).max()


TOL = {8: 1e-12, 4: 1e-5}


def rotate_links(gauge, H, eps):
    """QDP links exp(eps H) U for anti-Hermitian H [4][V][3][3]"""
    w, v = np.linalg.eigh(-1j * H)
    E = np.einsum("...ij,...j,...kj->...ik", v, np.exp(1j * eps * w), v.conj())
    U = E @ (gauge[..., 0] + 1j * gauge[..., 1])
    return np.stack([U.real, U.imag], -1)
