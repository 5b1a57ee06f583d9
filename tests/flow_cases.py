"""Cases shared by the CPU and GPU tiers of the gradient flow: one runner for the host twin (numpy) and the library (torch)
over b200_gauge_flow / b200_gauge_observables, the flow actions and the field builders."""
import ctypes as C

import numpy as np

import gauge_cases as GC
from quda_b200 import gauge as GP

EPS, STEPS = 0.02, 5
ACTIONS = sorted(GP.FLOW_ACTIONS)
SHAPES = GC.SHAPES + [(8, 8, 8, 8)]
FIELDS = {"near_identity": lambda X, s: GC.near_identity_links(X, s, 0.1), "haar": GC.haar_links}


class Runner(GC.Runner):
    """GC.Runner with the gradient flow and the observables"""

    def flow_rc(self, gauge, X, table, lengths, coeffs, n, max_length, eps, n_steps, prec=8, in_place=False):
        typ = np.float64 if prec == 8 else np.float32
        g = self._put(np.asarray(gauge, dtype=typ))
        out = g if in_place else self._put(np.zeros_like(np.asarray(gauge, dtype=typ)))
        t = np.ascontiguousarray(table, dtype=np.int32)
        rc = self._fn("gauge_flow")(self._links(out), self._links(g), (C.c_int * 4)(*X), prec, t.ctypes.data_as(C.POINTER(C.c_int)),
                                    (C.c_int * len(lengths))(*lengths), (C.c_double * len(coeffs))(*coeffs), n, max_length,
                                    float(eps), int(n_steps), None)
        return rc, self._get(out)

    def flow(self, gauge, X, action, eps=EPS, n_steps=STEPS, prec=8, in_place=False):
        paths, coeffs = GP.FLOW_ACTIONS[action] if isinstance(action, str) else action
        table, lengths, n, max_length = GP.path_table(paths)
        rc, out = self.flow_rc(gauge, X, table, lengths, coeffs, n, max_length, eps, n_steps, prec, in_place)
        self.check(rc)
        return out

    def observables(self, gauge, X, prec=8):
        """(energy (total, spatial, temporal), Q, density [V])"""
        g = self._put(np.asarray(gauge, dtype=np.float64 if prec == 8 else np.float32))
        dens = self._put(np.full(int(np.prod(X)), np.nan))
        e, q = (C.c_double * 3)(), C.c_double()
        self.check(self._fn("gauge_observables")(e, C.byref(q), self._ptr(dens), self._links(g), (C.c_int * 4)(*X), prec, None))
        return tuple(e), q.value, self._get(dens)


def flux_cases():
    """(planes of abelian_flux, sign of Q): the three pairings of the charge, (0,1)x(2,3) +, (0,2)x(1,3) -, (0,3)x(1,2) +"""
    return [(([(0, 1), 1], [(2, 3), 2]), 1), (([(0, 2), 2], [(1, 3), 1]), -1), (([(0, 3), 1], [(1, 2), 1]), 1)]


def flux_charge(phis, planes, sign):
    """Q = sign 2 n n' (sin phi / phi)(sin phi' / phi')"""
    (pa, na), (pb, nb) = planes
    a, b = phis[tuple(pa)], phis[tuple(pb)]
    return sign * 2 * na * nb * (np.sin(a) / a) * (np.sin(b) / b)


def flux_energy(phis):
    return 2 * sum(np.sin(p) ** 2 for p in phis.values())
