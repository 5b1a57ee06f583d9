"""GPU tier of the gauge half of an HMC step: libquda_b200 against the host twin bit for bit in fp64 and against the
reference's host gauge force / momentum action in both precisions; repeated calls bit-identical and the in-place update;
a two-flavour clover HMC trajectory whose driver lives here (gauge_force + compute_clover_force, update_gauge_field,
load_gauge and compute_clover_field after every link update): |dH| falls as dt^2, the trajectory is reversible, and the
force of the full update matches a finite difference of H computed by the library alone."""
import numpy as np
import pytest
import torch

import gauge_cases as G
from common import CudaMem, Problem
from gauge_twin import gauge_twin
from quda_b200 import dirac as DR
from quda_b200 import dslash as D
from quda_b200 import gauge as GP
from quda_b200 import lib as L

pytestmark = pytest.mark.gpu


def lib():
    return G.Runner(L.load(), "b200", dev=True)


def twin():
    return G.Runner(gauge_twin(), "twin")


@pytest.mark.parametrize("X", G.SHAPES + [(8, 8, 8, 8)])
@pytest.mark.parametrize("paths", G.PATH_SETS)
@pytest.mark.parametrize("field", sorted(G.FIELDS))
def test_library_matches_twin_and_reference(X, paths, field):
    V = int(np.prod(X))
    gauge = G.FIELDS[field](X, 11)
    mom0 = G.random_mom(V, 5, 0.1)
    p, c = G.path_set(paths)
    got = lib().force(mom0, gauge, X, p, c, 0.2)
    assert np.array_equal(got, twin().force(mom0, gauge, X, p, c, 0.2))
    assert np.array_equal(got, lib().force(mom0, gauge, X, p, c, 0.2))  # repeated calls: bit-identical
    got4 = lib().force(mom0, gauge, X, p, c, 0.2, prec=4)
    if G.have_ref():
        want = G.ref_force(mom0, gauge, X, p, c, 0.2)
        assert G.deviation(got, want, mom0) <= 1e-13
        assert G.deviation(got4, want, mom0) <= 1e-5
    assert G.deviation(got4, got, mom0) <= 1e-5
    for exact in (True, False):
        for conj in (False, True):
            u = lib().update(gauge, mom0 * 10, X, 0.3, conj, exact)
            assert np.array_equal(u, twin().update(gauge, mom0 * 10, X, 0.3, conj, exact))
            assert np.array_equal(u, lib().update(gauge, mom0 * 10, X, 0.3, conj, exact, in_place=True))
            assert np.abs(lib().update(gauge, mom0 * 10, X, 0.3, conj, exact, prec=4) - u).max() <= 2e-6
    for prec in (8, 4):
        m = mom0.astype(np.float64 if prec == 8 else np.float32)
        S = lib().mom_action(m, X, prec)
        assert S == lib().mom_action(m, X, prec)
        if prec == 8:
            assert S == twin().mom_action(m, X, prec)
        if G.have_ref():
            assert abs(S - G.ref_mom_action(m)) <= {8: 1e-12, 4: 1e-7}[prec] * np.abs(m).sum()
        pl = lib().plaquette(gauge, X, prec)
        assert pl == lib().plaquette(gauge, X, prec)
        if prec == 8:
            assert pl == twin().plaquette(gauge, X, prec)
        assert np.allclose(pl, G.plaquette(gauge, X), rtol=0, atol={8: 1e-14, 4: 1e-6}[prec])


def test_python_interface_in_place_and_device_load_gauge():
    X = (4, 6, 8, 10)
    V = int(np.prod(X))
    gauge = G.antiperiodic(G.haar_links(X, 3), X)
    mom0 = G.random_mom(V, 4, 0.5)
    g = torch.from_numpy(gauge).cuda()
    m = torch.from_numpy(mom0).cuda()
    out = GP.update_gauge_field(g, m, 0.2, X=X)
    want = twin().update(gauge, mom0, X, 0.2)
    assert np.array_equal(out.cpu().numpy(), want)
    same = GP.update_gauge_field(g, m, 0.2, X=X, out=g)
    assert same is g and np.array_equal(g.cpu().numpy(), want)
    p, c = G.path_set("plaq+rect")
    GP.gauge_force(m, g, p, c, 0.1, X=X)
    assert np.array_equal(m.cpu().numpy(), twin().force(mom0, want, X, p, c, 0.1))
    assert GP.mom_action(m) == twin().mom_action(m.cpu().numpy(), X)
    assert GP.plaquette(g, X=X) == twin().plaquette(want, X)
    # native links rebuilt from the device links equal those loaded from the same links on the host
    a = D.load_gauge(g, X, 8, 18, t_boundary=-1)
    b = D.load_gauge(want, X, 8, 18, t_boundary=-1)
    assert torch.equal(a.buf, b.buf)


# ------------------------------------------------------------------ a two-flavour clover HMC trajectory
KAPPA, CSW, BETA, TAU = 0.12, 1.3, 5.5, 0.5
X8 = (8, 8, 8, 8)
PLAQ, PLAQ_C = G.path_set("plaq")


class Hmc:
    """the driver: fp64, asymmetric even-even clover-PC operator, one pseudofermion phi = Mhat^+ eta (multiplicity 2)"""

    def __init__(self, seed=1):
        self.X, self.V = X8, int(np.prod(X8))
        self.P = Problem(self.X, 8, 18, CudaMem)
        gauge = G.antiperiodic(G.near_identity_links(self.X, seed, 0.1), self.X)
        self.U0 = torch.from_numpy(gauge).cuda()
        rng = np.random.default_rng(seed + 1)
        eta = rng.normal(size=(self.V // 2, 4, 3, 2)) * np.sqrt(0.5)
        op, _ = self.operator(self.U0)
        self.phi = self.P.empty(1)
        op.Mdag(self.phi, self.P.to_dev(eta))
        self.phi_h = self.P.to_host(self.phi)
        self.mom0 = torch.from_numpy(G.random_mom(self.V, seed + 2)).cuda()

    def operator(self, U):
        Un = D.load_gauge(U, self.X, 8, 18, t_boundary=-1)
        A, Ainv, trlog = D.compute_clover_field(U, self.X, 8, KAPPA, CSW)
        return DR.Dirac("cloverpc", Un, KAPPA, clover=A, clover_inv=Ainv, matpc_type=DR.MATPC_EVEN_EVEN_ASYMMETRIC), trlog

    def solve(self, U):
        op, trlog = self.operator(U)
        x = self.P.empty(1)
        p = DR.invert_multishift_cg(op, None, [x], self.phi, [0.0], tol=1e-12)
        assert p.true_res_offset[0] < 1e-11
        return op, x, trlog

    def action(self, U):
        """beta 6 V (1 - plaq) + phi^+ x - 2 tr log A_odd"""
        _, x, trlog = self.solve(U)
        return BETA * 6 * self.V * (1 - GP.plaquette(U, X=self.X)[0]) + float(np.sum(self.phi_h * self.P.to_host(x))) - 2 * trlog[1]

    def H(self, U, mom):
        return GP.mom_action(mom) + self.action(U)

    def kick(self, U, mom, eps):
        GP.gauge_force(mom, U, PLAQ, PLAQ_C, eps * BETA / 3, X=self.X)
        op, x, _ = self.solve(U)
        DR.compute_clover_force(mom, eps, [x], [1.0], KAPPA, CSW, 2, U, op)

    def leapfrog(self, U, mom, n):
        U, mom, dt = U.clone(), mom.clone(), TAU / n
        self.kick(U, mom, 0.5 * dt)
        for i in range(n):
            GP.update_gauge_field(U, mom, dt, X=self.X, out=U)
            self.kick(U, mom, dt if i < n - 1 else 0.5 * dt)
        return U, mom


@pytest.fixture(scope="module")
def hmc():
    return Hmc()


def test_hmc_energy_violation_falls_as_dt_squared(hmc):
    H0 = hmc.H(hmc.U0, hmc.mom0)
    dH = []
    for n in (5, 10, 20):
        U, mom = hmc.leapfrog(hmc.U0, hmc.mom0, n)
        dH.append(abs(hmc.H(U, mom) - H0))
    print("dH at 5, 10, 20 steps:", dH)
    for a, b in zip(dH, dH[1:]):
        assert 3.0 <= a / b <= 5.0, dH


def test_hmc_trajectory_is_reversible(hmc):
    H0 = hmc.H(hmc.U0, hmc.mom0)
    U1, m1 = hmc.leapfrog(hmc.U0, hmc.mom0, 10)
    U2, m2 = hmc.leapfrog(U1, -m1, 10)
    print("reversibility: links", float((U2 - hmc.U0).abs().max()), "H", abs(hmc.H(U2, -m2) - H0))
    assert float((U2 - hmc.U0).abs().max()) <= 1e-8
    assert abs(hmc.H(U2, -m2) - H0) <= 1e-6


def test_hmc_force_matches_finite_difference_of_H(hmc):
    """sum_links tr(H F) with F = (mom after one kick of size dt - mom before) / dt against dS/d eps along U -> exp(eps H) U,
    the rotation done by update_gauge_field and S evaluated by the library"""
    dt = 0.5
    mom = torch.zeros_like(hmc.mom0)
    hmc.kick(hmc.U0, mom, dt)
    import clover_force_ref as CF
    Fm = CF.mom_to_matrices(mom.cpu().numpy()) / dt
    Hd = torch.from_numpy(G.random_mom(hmc.V, 99)).cuda()
    Hm = CF.mom_to_matrices(Hd.cpu().numpy())  # [V][4][3][3]
    predicted = np.einsum("vmij,vmji->", Hm, Fm).real
    eps = 1e-3
    S = {k: hmc.action(GP.update_gauge_field(hmc.U0, Hd, k * eps, X=hmc.X)) for k in (2, 1, -1, -2)}
    fd = (8 * (S[1] - S[-1]) - (S[2] - S[-2])) / (12 * eps)
    print("finite difference", fd, "predicted", predicted)
    assert abs(fd - predicted) <= 1e-6 * abs(fd), (fd, predicted)
