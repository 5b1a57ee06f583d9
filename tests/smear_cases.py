"""Cases shared by the CPU and GPU tiers of gauge smearing: one runner for the host twin (numpy) and the library (torch)
over b200_gauge_smear, the typical coefficients of each kind, and the shapes and fields of the flow tests."""
import ctypes as C

import numpy as np

import flow_cases as FC
import gauge_cases as GC
import smear_twin as ST
from quda_b200 import gauge as GP

# typical parameters: APE alpha = 0.6, stout rho = 0.1, over-improved rho = 0.06 with eps = -0.25, HYP (0.75, 0.6, 0.3)
COEFFS = {"ape": {"alpha": 0.6}, "stout": {"rho": 0.1}, "ovrimp_stout": {"rho": 0.06, "epsilon": -0.25},
          "hyp": {"alpha1": 0.75, "alpha2": 0.6, "alpha3": 0.3}}
KINDS = sorted(COEFFS)
IGNORE = [-1, 0, 1, 2, 3]
SHAPES = FC.SHAPES
FIELDS = FC.FIELDS
STEPS = 3


def coeff_array(kind, coeffs=None):
    c = coeffs or COEFFS[kind]
    return [float(c[n]) for n in GP.SMEAR_KINDS[kind][1]]


class Runner(FC.Runner):
    """FC.Runner with b200_gauge_smear"""

    def smear_rc(self, gauge, X, type_, coeff, dir_ignore, n_steps, prec=8, in_place=False):
        typ = np.float64 if prec == 8 else np.float32
        g = self._put(np.asarray(gauge, dtype=typ))
        out = g if in_place else self._put(np.full(np.shape(gauge), np.nan, dtype=typ))
        c = (C.c_double * 3)(*(list(coeff) + [0.0] * (3 - len(coeff))))
        rc = self._fn("gauge_smear")(self._links(out), self._links(g), (C.c_int * 4)(*X), prec, type_, c, int(dir_ignore),
                                     int(n_steps), None)
        return rc, self._get(out)

    def smear(self, gauge, X, kind, n_steps=STEPS, dir_ignore=-1, prec=8, in_place=False, coeffs=None):
        rc, out = self.smear_rc(gauge, X, GP.SMEAR_KINDS[kind][0], coeff_array(kind, coeffs), dir_ignore, n_steps, prec, in_place)
        self.check(rc)
        return out


def twin():
    return Runner(ST.smear_twin(), "twin")


def time_slice_sites(X, t):
    """parity-major indices of the sites with x_3 = t"""
    from quda_b200 import fields as F
    idx = []
    for p in range(2):
        c = F.cb_coords(X, p)
        idx.append(p * len(c) + np.nonzero(c[:, 3] == t)[0])
    return np.concatenate(idx)


def su3_deviation(gauge):
    """(max |U^+ U - 1|, max |det U - 1|) over the links"""
    U = GC.cplx(gauge)
    uu = np.einsum("...ki,...kj->...ij", U.conj(), U) - np.eye(3)
    return float(np.abs(uu).max()), float(np.abs(np.linalg.det(U) - 1).max())
