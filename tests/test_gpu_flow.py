"""GPU tier of the gradient flow and its observables: libquda_b200 against the host twin bit for bit in fp64 and fp32 (links,
E, Q and the charge density), on the CPU tier's shapes and 16^3x32; the finite-difference, abelian-flux and symmetry checks
again through quda_b200.gauge on device tensors, in place and out of place; and the flow of the end configuration of a short
clover HMC trajectory to t = 1."""
import numpy as np
import pytest
import torch

import flow_cases as FC
import flow_ref as FR
import gauge_cases as GC
from flow_twin import flow_twin
from quda_b200 import gauge as GP
from quda_b200 import lib as L

pytestmark = pytest.mark.gpu


def lib():
    return FC.Runner(L.load(), "b200", dev=True)


def twin():
    return FC.Runner(flow_twin(), "twin")


@pytest.mark.parametrize("X", FC.SHAPES)
@pytest.mark.parametrize("action", FC.ACTIONS)
@pytest.mark.parametrize("field", sorted(FC.FIELDS))
def test_library_matches_twin(X, action, field):
    gauge = FC.FIELDS[field](X, 31)
    for prec in (8, 4):
        got = lib().flow(gauge, X, action, prec=prec)
        assert np.array_equal(got, twin().flow(gauge, X, action, prec=prec))
        assert np.array_equal(got, lib().flow(gauge, X, action, prec=prec))  # repeated calls
        assert np.array_equal(got, lib().flow(gauge, X, action, prec=prec, in_place=True))
        e, q, dens = lib().observables(got, X, prec)
        et, qt, denst = twin().observables(got, X, prec)
        assert e == et and q == qt and np.array_equal(dens, denst)
        assert lib().observables(got, X, prec)[:2] == (e, q)


@pytest.mark.parametrize("action", FC.ACTIONS)
def test_library_matches_twin_16x16x16x32(action):
    X = (16, 16, 16, 32)
    gauge = GC.haar_links(X, 5)
    for prec in (8, 4):
        got = lib().flow(gauge, X, action, n_steps=1, prec=prec)
        assert np.array_equal(got, twin().flow(gauge, X, action, n_steps=1, prec=prec))
        e, q, dens = lib().observables(got, X, prec)
        et, qt, denst = twin().observables(got, X, prec)
        assert e == et and q == qt and np.array_equal(dens, denst)


# ------------------------------------------------------------------ the checks through quda_b200.gauge
def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("action", FC.ACTIONS)
def test_finite_difference_through_python(action):
    X = (4, 6, 8, 10)
    gauge = GC.haar_links(X, 12)
    g = dev(gauge)
    paths, coeffs = GP.FLOW_ACTIONS[action]
    h = 1e-3
    S = {k: FR.action(GP.gradient_flow(g, k * h, 1, X=X, action=action)[0].cpu().numpy(), X, paths, coeffs)
         for k in (2, 1, -1, -2)}
    fd = (8 * (S[1] - S[-1]) - (S[2] - S[-2])) / (12 * h)
    V = int(np.prod(X))
    m = torch.zeros((V, 4, 10), dtype=torch.float64, device="cuda")
    GP.gauge_force(m, g, paths, coeffs, 1.0, X=X)
    want = -2 * (GP.mom_action(m, X=X) + 16 * V)
    print(action, "dS/dt", fd, "-sum |TA(Omega)|^2", want)
    assert abs(fd - want) <= 1e-8 * abs(want)


@pytest.mark.parametrize("case", range(3))
def test_abelian_flux_through_python(case):
    X = (4, 6, 8, 10)
    planes, sign = FC.flux_cases()[case]
    gauge, phis = FR.abelian_flux(X, planes)
    g = dev(gauge)
    for action in FC.ACTIONS:
        f, rows = GP.gradient_flow(g, FC.EPS, FC.STEPS, X=X, action=action, meas_interval=FC.STEPS)
        assert float((f - g).abs().max()) <= 1e-14 and len(rows) == 2
    dens = torch.empty(int(np.prod(X)), dtype=torch.float64, device="cuda")
    o = GP.gauge_observables(g, X=X, density=dens)
    assert abs(o["energy"][0] - FC.flux_energy(phis)) <= 1e-13 * FC.flux_energy(phis)
    assert abs(o["qcharge"] - FC.flux_charge(phis, planes, sign)) <= 1e-12
    assert abs(float(dens.sum()) - o["qcharge"]) <= 1e-12 * float(dens.abs().sum())
    flipped = [[planes[0][0], -planes[0][1]], planes[1]]
    assert abs(GP.gauge_observables(dev(FR.abelian_flux(X, flipped)[0]), X=X)["qcharge"] + o["qcharge"]) <= 1e-12


@pytest.mark.parametrize("action", FC.ACTIONS)
def test_symmetries_through_python(action):
    X = (4, 6, 8, 10)
    gauge = GC.haar_links(X, 8)
    gt = FR.random_su3((X[3], X[2], X[1], X[0]), 9)
    g, g2 = dev(gauge), dev(FR.gauge_transform(gauge, X, gt))
    o, o2 = GP.gauge_observables(g, X=X), GP.gauge_observables(g2, X=X)
    dens = torch.empty(int(np.prod(X)), dtype=torch.float64, device="cuda")
    GP.gauge_observables(g, X=X, density=dens)
    qs = float(dens.abs().sum())
    assert np.allclose(o2["energy"], o["energy"], rtol=1e-12, atol=0) and abs(o2["qcharge"] - o["qcharge"]) <= 1e-12 * qs
    assert np.allclose(o2["plaquette"], o["plaquette"], rtol=1e-12, atol=0)
    f = GP.gradient_flow(g, FC.EPS, FC.STEPS, X=X, action=action)[0].cpu().numpy()
    f2 = GP.gradient_flow(g2, FC.EPS, FC.STEPS, X=X, action=action)[0].cpu().numpy()
    assert np.abs(f2 - FR.gauge_transform(f, X, gt)).max() <= 1e-12
    # reflection in x flips Q and keeps E
    r = GP.gauge_observables(dev(FR.reflect_x(gauge, X)), X=X)
    assert np.allclose(r["energy"], o["energy"], rtol=1e-12, atol=0) and abs(r["qcharge"] + o["qcharge"]) <= 1e-12 * qs
    # the boundary sign is carried bit for bit; out = in flows in place
    ga = dev(GC.antiperiodic(gauge, X))
    fa, _ = GP.gradient_flow(ga, FC.EPS, FC.STEPS, X=X, action=action)
    assert np.array_equal(fa.cpu().numpy(), GC.antiperiodic(f, X))
    same, _ = GP.gradient_flow(ga, FC.EPS, FC.STEPS, X=X, action=action, out=ga)
    assert same is ga and torch.equal(ga, fa)


# ------------------------------------------------------------------ the end of an HMC trajectory, flowed to t = 1
def test_flow_of_an_hmc_configuration():
    from test_gpu_gauge import X8, Hmc
    hmc = Hmc()
    U, _ = hmc.leapfrog(hmc.U0, hmc.mom0, 10)
    flowed, rows = GP.gradient_flow(U, 0.01, 100, X=X8, action="wilson", meas_interval=10)
    for t, plaq, energy, q in rows:
        print(f"t {t:5.2f}  plaquette {plaq[0]:.12f}  E {energy[0]:.10f}  t^2 E {t * t * energy[0]:.8f}  Q {q:+.6f}")
    assert [r[0] for r in rows] == pytest.approx([0.1 * k for k in range(11)])
    plaq = [r[1][0] for r in rows]
    assert all(b > a for a, b in zip(plaq, plaq[1:]))
    assert torch.equal(flowed, GP.gradient_flow(U, 0.01, 100, X=X8, action="wilson")[0])
